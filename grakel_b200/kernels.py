"""Estimator classes of the hot path, mirroring the reference's operator API.

Same class names, constructor signatures, method names and error behaviour as
grakel.kernels.{Kernel, WeisfeilerLehman, VertexHistogram, ShortestPath,
ShortestPathAttr} (kernel.py:23-456, weisfeiler_lehman.py:23-555,
vertex_histogram.py:23-219, shortest_path.py:16-515), but every kernel matrix is
produced by the CUDA engine behind `grakel_b200._lib` -- there is no CPU path.

Fitted state is host-resident numpy / Python objects (a packed CSR `Block` and
the level-0 label dictionary), so fitted estimators pickle like the reference's
(grakel/tests/test_common.py:53-58); device buffers are re-created on demand.
"""
from __future__ import annotations

import contextlib
import copy
import math
import functools
import warnings
from collections.abc import Iterable
from collections import Counter
from itertools import chain, filterfalse
from numbers import Real
import time

import numpy as np
from scipy.special import binom
from sklearn.base import BaseEstimator, TransformerMixin
from sklearn.exceptions import NotFittedError
from sklearn.utils import check_random_state
from sklearn.utils.validation import check_is_fitted

from . import _lib
from .packing import Block, Graph, adjacency_and_order, label_ids, pack


class Fitted:
    """What `fit` keeps: the packed graphs, their level-0 label ids, the label dictionary.  Under a relabelling
    framework also `skip`, the vertices absent from the levels >= 1 (HadamardCode), and the base kernel's own data:
    its graphs (`base`, _WlBaseData) or its per-level embeddings (`pm`, _PmData)."""

    base = None
    pm = None

    def __init__(self, block, ids, dictionary=None, skip=None):
        self.block = block
        self.ids = ids
        self.dictionary = dictionary
        self.skip = skip

    def __len__(self):
        return self.block.n_graphs

    @staticmethod
    def concat(a, b):
        """The fitted input `a` followed by a transform's `b`: what one joint device run reads."""
        skip = None
        if a.skip is not None or b.skip is not None:
            fa = a.skip if a.skip is not None else np.zeros(a.block.n_vertices, dtype=bool)
            fb = b.skip if b.skip is not None else np.zeros(b.block.n_vertices, dtype=bool)
            skip = np.concatenate([fa, fb])
        out = Fitted(Block.concat(a.block, b.block), np.concatenate([a.ids, b.ids]), a.dictionary, skip)
        if a.base is not None:
            out.base = _WlBaseData.concat(a.base, b.base)
        if a.pm is not None:
            out.pm = _PmData.concat(a.pm, b.pm)
        return out


class CoreLevel:
    """One core level of a CoreFramework fold (core_framework.py): while it is set as a base kernel's `_core_level`,
    the kernel's runs use the fold's engine, and a run that produces K adds it into the device-resident sum at `rows`
    (its rows) and `cols` (its fitted columns) instead of returning it; the fold's seconds add up in times["fold"]."""

    def __init__(self, eng, level, rows, cols, times):
        self.eng, self.level, self.rows, self.cols, self.times = eng, level, rows, cols, times


def _run_engine(est):
    lvl = getattr(est, "_core_level", None)
    return _lib.engine(getattr(est, "device_", None)) if lvl is None else contextlib.nullcontext(lvl.eng)


def _gram_or_fold(est, eng, n_graphs, n_fit, want_matrix=True, want_diag=True, stats=None, **kw):
    """eng.gram, or for a CoreFramework level the fold of its K (the base kernels run un-normalised there)."""
    lvl = getattr(est, "_core_level", None)
    if lvl is None or not want_matrix:
        return eng.gram(n_graphs, n_fit=n_fit, out=None if want_matrix else False, want_diag=want_diag, stats=stats,
                        **kw)
    t = time.perf_counter()
    xd, yd = eng.core_level_add(lvl.level, n_fit, lvl.rows, lvl.cols, n_graphs, want_diag=want_diag, stats=stats)
    lvl.times["fold"] += time.perf_counter() - t
    return None, xd, yd


class Kernel(BaseEstimator, TransformerMixin):
    """Estimator contract of grakel.kernels.Kernel (kernel.py:23-456).

    Subclasses provide `parse_input` (host packing) and `_device_features`
    (which feature kernel to run); fit / transform / fit_transform / diagonal /
    set_params behave as in the reference."""

    X = None
    _graph_format = "dictionary"
    _method_calling = 0
    _nan_to_num = False

    def __init__(self, n_jobs=None, normalize=False, verbose=False):
        self.verbose = verbose
        self.n_jobs = n_jobs
        self.normalize = normalize
        self._initialized = dict(n_jobs=False)

    # ---- reference protocol --------------------------------------------------
    def fit(self, X, y=None):
        self._is_transformed = False
        self._method_calling = 1
        self.initialize()
        if X is None:
            raise ValueError("`fit` input cannot be None")
        self.X = self.parse_input(X)
        return self

    def transform(self, X):
        self._method_calling = 3
        check_is_fitted(self, ["X"])
        if X is None:
            raise ValueError("`transform` input cannot be None")
        Y = self.parse_input(X)
        K, xdiag, ydiag = self._run(Block.concat(self.X.block, Y.block), np.concatenate([self.X.ids, Y.ids]),
                                    n_fit=self.X.block.n_graphs)
        self._X_diag = xdiag  # kernel.py:160-164 computes it on demand; the joint run returns it anyway
        self._Y_diag = ydiag
        self._is_transformed = True
        if self.normalize:
            self._warn_unnormalizable(self._X_diag, ydiag)
        return K

    def fit_transform(self, X, y=None):
        self._method_calling = 2
        self.fit(X)
        K, xdiag, _ = self._run(self.X.block, self.X.ids, n_fit=self.X.block.n_graphs)
        self._X_diag = xdiag
        if self.normalize:
            self._warn_unnormalizable(xdiag)
        return K

    def diagonal(self):
        check_is_fitted(self, ["X"])
        try:
            check_is_fitted(self, ["_X_diag"])
        except NotFittedError:
            _, self._X_diag, _ = self._run(self.X.block, self.X.ids, n_fit=self.X.block.n_graphs, want_matrix=False)
        if getattr(self, "_is_transformed", False):
            return self._X_diag, self._Y_diag
        return self._X_diag

    def _warn_unnormalizable(self, *diagonals):
        """kernel.py:206-234: say why a normalised matrix contains NaNs."""
        name = type(self).__name__
        for d in diagonals:
            d = np.asarray(d, dtype=float)
            if np.any(d == 0):
                warnings.warn(name + " has zero self similarities, so normalizing it yields NaNs: those graphs "
                              "have no features this kernel can see. Either drop them or pass normalize=False.",
                              RuntimeWarning)
                break

    def initialize(self):
        """kernel.py:386-399.  `n_jobs` is validated and then ignored: the whole Gram
        matrix is one device job (ShortestPath already ignores it, shortest_path.py:239-242)."""
        if not self._initialized["n_jobs"]:
            if type(self.n_jobs) is not int and self.n_jobs is not None:
                raise ValueError("n_jobs parameter must be an int indicating the number of jobs as in joblib or None")
            self._parallel = None
            self._initialized["n_jobs"] = True

    def parse_input(self, X):
        raise NotImplementedError

    def pairwise_operation(self, x, y):
        raise NotImplementedError("Pairwise operation is not implemented!")

    # ---- generic pairwise driver (kernel.py:236-296, 298-336) ---------------------
    # For kernels whose value needs a per-pair Python callback (ShortestPathAttr with a user metric): `self.X` is then
    # a plain list of per-graph items produced on the device and the matrix is filled pair by pair on the host, in the
    # reference's order and with its symmetrisation.  The Gram kernels never take this route.
    def _calculate_kernel_matrix(self, Y=None):
        if Y is None:
            n = len(self.X)
            K = np.zeros(shape=(n, n))
            cache = []
            for i, x in enumerate(self.X):
                K[i, i] = self.pairwise_operation(x, x)
                for j, y in enumerate(cache):
                    K[j, i] = self.pairwise_operation(y, x)
                cache.append(x)
            return np.triu(K) + np.triu(K, 1).T
        K = np.zeros(shape=(len(Y), len(self.X)))
        for j, y in enumerate(Y):
            for i, x in enumerate(self.X):
                K[j, i] = self.pairwise_operation(y, x)
        return K

    def _pairwise_fit_transform(self, X):
        self._method_calling = 2
        self.fit(X)
        km = self._calculate_kernel_matrix()
        self._X_diag = np.diagonal(km).copy()
        if self.normalize:  # kernel.py:196-203
            self._warn_unnormalizable(self._X_diag)
            with np.errstate(invalid="ignore", divide="ignore"):
                km = km / np.sqrt(np.outer(self._X_diag, self._X_diag))
        return km

    def _pairwise_transform(self, X):
        self._method_calling = 3
        check_is_fitted(self, ["X"])
        if X is None:
            raise ValueError("`transform` input cannot be None")
        Y = self.parse_input(X)
        km = self._calculate_kernel_matrix(Y)
        self._Y = Y
        self._is_transformed = True
        if self.normalize:  # kernel.py:155-164
            X_diag, Y_diag = self._pairwise_diagonal()
            self._warn_unnormalizable(X_diag, Y_diag)
            with np.errstate(invalid="ignore", divide="ignore"):
                km /= np.sqrt(np.outer(Y_diag, X_diag))
        return km

    def _pairwise_diagonal(self):
        check_is_fitted(self, ["X"])
        try:
            check_is_fitted(self, ["_X_diag"])
        except NotFittedError:
            self._X_diag = np.array([self.pairwise_operation(x, x) for x in self.X], dtype=float)
        if getattr(self, "_is_transformed", False) and hasattr(self, "_Y"):
            self._Y_diag = np.array([self.pairwise_operation(y, y) for y in self._Y], dtype=float)
            return self._X_diag, self._Y_diag
        return self._X_diag

    def set_params(self, **params):
        """kernel.py:417-433: a changed parameter is re-validated at the next fit."""
        if len(self._initialized):
            params = copy.deepcopy(params)
            for key in params:
                key, delim, sub_key = key.partition("__")
                if delim:
                    if sub_key in self._initialized:
                        self._initialized[sub_key] = False
                elif key in self._initialized:
                    self._initialized[key] = False
        super().set_params(**params)
        return self

    # ---- device side ---------------------------------------------------------
    def _device_features(self, engine):
        raise NotImplementedError

    def _run(self, block, ids, n_fit, want_matrix=True):
        """pack -> feature kernels -> Gram, all on the device.  Returns (K, xdiag, ydiag)."""
        with _run_engine(self) as eng:
            eng.pack(block.graph_ptr, block.row_ptr, block.col_idx, ids, block.weights, block.attrs)
            self.stats_ = self._device_features(eng)
            K, xd, yd = _gram_or_fold(self, eng, block.n_graphs, n_fit, want_matrix,
                                      normalize=bool(self.normalize) and want_matrix, nan_to_num=self._nan_to_num,
                                      stats=self.stats_)
        if self.verbose:
            print(type(self).__name__, self.stats_.as_dict())
        return K, xd, yd


# ------------------------------------------------------------------------------
class VertexHistogram(Kernel):
    """Vertex histogram kernel (vertex_histogram.py:23-219): K = Phi Phi^T with
    Phi[g, l] = number of vertices of g carrying label l."""

    def __init__(self, n_jobs=None, normalize=False, verbose=False, sparse="auto"):
        super().__init__(n_jobs=n_jobs, normalize=normalize, verbose=verbose)
        self.sparse = sparse
        self._initialized.update({"sparse": True})

    def parse_input(self, X):
        from .packing import iter_elements
        if self._method_calling in (1, 2):
            known = None
        else:
            known = self.X.dictionary
        if isinstance(X, Block):  # packed input (datasets.read_tu): only the label multisets matter
            X.require("wl")
            block = Block(X.graph_ptr, np.zeros(X.n_vertices + 1, dtype=np.int64), np.zeros(0, dtype=np.int64), None,
                          X.labels)
            labels = X.labels
        else:
            sizes, labels = [0], []
            for _, _g, L in iter_elements(X, lambda n: n in (2, 3)):
                vals = list(L.values())
                labels.extend(vals)
                sizes.append(sizes[-1] + len(vals))
            if len(sizes) == 1:
                raise ValueError("parsed input is empty")
            block = Block(np.asarray(sizes), np.zeros(sizes[-1] + 1, dtype=np.int64), np.zeros(0, dtype=np.int64),
                          None, labels)
        if known is None:
            ids, new = label_ids(labels, None, sort_new=False)
            dictionary = new
            self.sparse_ = True
        else:
            ids, new = label_ids(labels, known, sort_new=False)
            dictionary = known
        return Fitted(block, ids, dictionary)

    def _device_features(self, eng):
        return eng.wl_features(0)


# ------------------------------------------------------------------------------
def _path_sum_order(block, algorithm_type):
    """Which of the reference's two shortest-path algorithms defines the path sums of a block with real-valued
    weights: "auto" runs Floyd-Warshall on adjacency input and Dijkstra on edge dictionaries (shortest_path.py:244-252,
    graph.py:652-656), and the two round differently (SURVEY 7).  Returns True for Dijkstra's order.  Integer-valued
    weights give the same distances either way."""
    if block.weights is None or not np.any(block.weights != np.rint(block.weights)):
        return False
    if algorithm_type == "floyd_warshall":
        return False
    if algorithm_type == "dijkstra":
        return True
    if block.all_adjacency:
        return False
    if getattr(block, "any_adjacency", False):
        raise NotImplementedError("real-valued edge weights with adjacency and dictionary inputs mixed in one call: the "
                                  "reference would use a different algorithm per graph; pass algorithm_type explicitly")
    return True


def _edge_label_values(X):
    """Edge-label values per element, with the element checks of EdgeHistogram.parse_input
    (edge_histogram.py:76-103): elements must have exactly three members (graph, node labels,
    edge labels) or be `Graph` objects; only the VALUES of the edge-label dictionary are used."""
    if not isinstance(X, Iterable):
        raise TypeError("input must be an iterable\n")
    out = []
    for idx, x in enumerate(iter(X)):
        if isinstance(x, Graph):
            if not x.edge_labels:
                raise ValueError("Graph does not have any labels for edges.")
            L = x.edge_labels
        else:
            is_iter = isinstance(x, Iterable)
            if is_iter:
                x = list(x)
            if not (is_iter and len(x) in (0, 3)):
                raise TypeError("each element of X must be either a graph object or a list with at least a graph like "
                                "object and node labels dict \n")
            if len(x) == 0:
                warnings.warn("Ignoring empty element on index: " + str(idx))
                continue
            L = x[2]
        out.append(list(L.values()))
    if not out:
        raise ValueError("parsed input is empty")
    return out


class EdgeHistogram(Kernel):
    """Edge histogram kernel (edge_histogram.py:23-212): K = Phi Phi^T with
    Phi[g, l] = number of edge-label entries of g equal to l.  On the device this is the
    vertex-histogram path over a block whose "vertices" are the edge-label entries."""

    _levels = 0

    def __init__(self, n_jobs=None, normalize=False, verbose=False, sparse="auto"):
        super().__init__(n_jobs=n_jobs, normalize=normalize, verbose=verbose)
        self.sparse = sparse
        self._initialized.update({"sparse": True})

    def initialize(self):
        if not self._initialized["n_jobs"]:  # edge_histogram.py:48-52
            if self.n_jobs is not None:
                warnings.warn("no implemented parallelization for EdgeHistogram")
            self._initialized["n_jobs"] = True

    def parse_input(self, X):
        values = _edge_label_values(X)
        sizes = np.concatenate([[0], np.cumsum([len(v) for v in values])])
        labels = [l for v in values for l in v]
        block = Block(sizes, np.zeros(int(sizes[-1]) + 1, dtype=np.int64), np.zeros(0, dtype=np.int64), None, labels)
        if self._method_calling in (1, 2):
            ids, dictionary = label_ids(labels, None, sort_new=False)
            self._labels = dictionary
            self.sparse_ = True
            return Fitted(block, ids, dictionary)
        ids, _ = label_ids(labels, self.X.dictionary, sort_new=False)
        return Fitted(block, ids, self.X.dictionary)

    def _device_features(self, eng):
        return eng.wl_features(self._levels)


# ------------------------------------------------------------------------------
class _LevelDictionaries(dict):
    """`_inv_labels` of a fitted WL estimator (weisfeiler_lehman.py:208-257): level 0 is built on the host by `fit`;
    the dictionaries of the levels >= 1 -- credential string -> compressed label, in the reference's own numbering --
    are exported from the device relabelling the first time one of them is asked for."""

    def __init__(self, level0, owner):
        super().__init__({0: level0})
        self._owner = owner

    def __missing__(self, level):
        owner = self._owner
        if owner is None or type(level) is not int or not 0 < level < owner._n_iter:
            raise KeyError(level)
        self.update(owner._export_level_dictionaries())
        return dict.__getitem__(self, level)

    def __reduce__(self):  # pickles as what has been materialised plus the owner
        return (_restore_level_dictionaries, (dict(self), self._owner))


def _restore_level_dictionaries(content, owner):
    d = _LevelDictionaries(content.get(0), owner)
    d.update(content)
    return d


def wl_reference_dictionaries(row_ptr, col_idx, level0_ids, n_level0, classes, n_fit_vertices=None):
    """The reference's per-level label dictionaries from the device partition.

    `classes[i]` (i >= 1) holds one class id per vertex (any numbering; `gk_wl_labels`).  The reference names a
    class by the string  str(own label) + "," + str(sorted neighbour labels)  over the labels of level i-1, sorts the
    distinct strings and numbers them on from where the previous level stopped (weisfeiler_lehman.py:223-246).
    One string per CLASS is built here (from the class's first vertex), not one per vertex.

    With `n_fit_vertices`, the block is the fitted graphs' vertices followed by a transform's (the joint partition of
    both): the classes the fitted vertices have are numbered as in the fit, the others in sorted order after them, and
    the next level again starts where the fit's did (weisfeiler_lehman.py:434-466).  Only the fitted classes enter the
    dictionaries then.
    Returns ({level: {credential: label}}, [reference label of every vertex, per level])."""
    prev = np.asarray(level0_ids, dtype=np.int64)
    count = int(n_level0)
    nfv = len(prev) if n_fit_vertices is None else int(n_fit_vertices)
    out, labels = {}, [prev]
    for i in range(1, len(classes)):
        uniq, first, inv = np.unique(np.asarray(classes[i]), return_index=True, return_inverse=True)
        inv = inv.reshape(-1)
        creds = []
        for v in first.tolist():
            nb = prev[col_idx[row_ptr[v]:row_ptr[v + 1]]]
            creds.append(str(int(prev[v])) + "," + str(sorted(nb.tolist())))
        if len(set(creds)) != len(creds):
            raise RuntimeError("two classes of level %d share a signature: the device partition is not the "
                               "reference's" % i)
        fitted = np.zeros(len(uniq), dtype=bool)
        fitted[inv[:nfv]] = True
        fit_k = [k for k in range(len(creds)) if fitted[k]]
        new_k = [k for k in range(len(creds)) if not fitted[k]]
        order = sorted(fit_k, key=creds.__getitem__) + sorted(new_k, key=creds.__getitem__)
        new_id = np.empty(len(uniq), dtype=np.int64)
        new_id[order] = count + np.arange(len(uniq), dtype=np.int64)
        out[i] = {creds[k]: count + r for r, k in enumerate(order[:len(fit_k)])}
        prev = new_id[inv]
        labels.append(prev)
        count += len(fit_k)
    return out, labels


# ------------------------------------------------------------------------------
_WL_GRAPH_BASES = ()  # set after the base classes: the bases whose WL route needs the list of graphs
_HC_GRAPH_BASES = ()  # ... and those of HadamardCode's per-level routes


def parse_base_kernel(est, default, allowed, refusal, check=None, copy=False):
    """(base, params) of a framework estimator's `base_graph_kernel`, checked as the reference checks it
    (weisfeiler_lehman.py:77-109, hadamard_code.py:68-97, core_framework.py:59-88): None (the framework's `default`),
    a Kernel class or (Kernel class, params dict), `normalize` dropped from the params.  A base outside `allowed`
    raises NotImplementedError(refusal); `check(base, params)` then runs the base kernel's own checks.  The params get
    the reference's normalize=False, the estimator's verbose and n_jobs=None; they are the caller's dict, edited in
    place as the reference does, unless `copy`."""
    base = est.base_graph_kernel
    if base is None:
        base, params = default, dict()
    elif type(base) is type and issubclass(base, Kernel):
        params = dict()
    else:
        try:
            base, params = base
        except Exception:
            raise TypeError("Base kernel was not formulated in the correct way. Check documentation.")
        if not (type(base) is type and issubclass(base, Kernel)):
            raise TypeError("The first argument must be a valid grakel.kernel.kernel Object")
        if type(params) is not dict:
            raise ValueError("If the second argument of base kernel exists, it must be a dictionary between "
                             "parameters names and values")
        if copy:
            params = dict(params)
        params.pop("normalize", None)
    if base not in allowed:
        raise NotImplementedError(refusal)
    if check is not None:
        check(base, params)
    params["normalize"] = False
    params["verbose"] = est.verbose
    params["n_jobs"] = None
    return base, params


def level_base_check(est, who, base, params, reads, ignores, copies):
    """The base kernel's own checks under a relabelling framework `est` (named `who`), and its refusals: a custom
    SubgraphMatching vertex kernel (it would read the framework's `reads` per level), ShortestPath(with_labels=False)
    (it ignores the framework's `ignores`: `copies` * ShortestPath is the same kernel).  Sets est._sm, the
    SubgraphMatching that checks the elements, or None."""
    est._sm = None
    if base is NeighborhoodSubgraphPairwiseDistance:
        NeighborhoodSubgraphPairwiseDistance(**{k: v for k, v in params.items() if k in ("r", "d")}).initialize()
    if base is OddSth:
        OddSth(h=params.get("h")).initialize()
    if base is SubgraphMatching:  # subgraph_matching.py:70-120
        sm = SubgraphMatching(**{k: v for k, v in params.items() if k in ("k", "kv", "ke", "lw")})
        sm.initialize()
        if sm.kv is not None and sm.kv is not _dirac:
            raise NotImplementedError("%s over SubgraphMatching runs kv=_dirac or kv=None: a custom vertex kernel "
                                      "reads the reference's %s per level" % (who, reads))
        est._sm = sm
    if base is PyramidMatch:  # pyramid_match.py:62-81
        PyramidMatch(**{k: v for k, v in params.items() if k in ("with_labels", "L", "d")}).initialize()
    if base is ShortestPath:
        if not params.get("with_labels", True):
            raise NotImplementedError("%s over ShortestPath(with_labels=False) ignores the %s; use %s * "
                                      "ShortestPath(with_labels=False)" % (who, ignores, copies))
        if params.get("algorithm_type", "auto") not in ("auto", "floyd_warshall", "dijkstra"):
            raise ValueError('Unsupported "algorithm_type"')


class WeisfeilerLehman(Kernel):
    """Weisfeiler-Lehman subtree kernel (weisfeiler_lehman.py:23-555).

    K = sum over levels 0..n_iter of the base kernel on the level's compressed
    labels.  The base kernels that run on the device: VertexHistogram (the
    subtree kernel, the reference default), EdgeHistogram, ShortestPath,
    PyramidMatch, NeighborhoodSubgraphPairwiseDistance, OddSth and
    SubgraphMatching.  Over NSPD and OddSth every level's labels are numbered
    the reference's way on the host (they read label numbers, not only the
    partition); OddSth's levels share one DAG pass and one exact Gram, NSPD's
    levels are folded one by one into a device-resident sum added in level
    order (DESIGN 4.21).  SubgraphMatching (kv `_dirac` or None) needs only the
    device partition: one clique enumeration gives every level's counts
    (DESIGN 4.23)."""

    _graph_format = "dictionary"
    _nan_to_num = True

    def __init__(self, n_jobs=None, verbose=False, normalize=False, n_iter=5, base_graph_kernel=VertexHistogram):
        super().__init__(n_jobs=n_jobs, verbose=verbose, normalize=normalize)
        self.n_iter = n_iter
        self.base_graph_kernel = base_graph_kernel
        self._initialized.update({"n_iter": False, "base_graph_kernel": False})
        self._base_graph_kernel = None

    def initialize(self):
        super().initialize()
        if not self._initialized["base_graph_kernel"]:  # weisfeiler_lehman.py:77-109
            self._base_graph_kernel, self._params = parse_base_kernel(
                self, VertexHistogram, (VertexHistogram, EdgeHistogram, ShortestPath, PyramidMatch,
                                        NeighborhoodSubgraphPairwiseDistance, OddSth, SubgraphMatching),
                "grakel_b200 runs WeisfeilerLehman over VertexHistogram (the subtree kernel), EdgeHistogram, "
                "ShortestPath, PyramidMatch, NeighborhoodSubgraphPairwiseDistance, OddSth or SubgraphMatching; other "
                "base kernels are outside the device hot path",
                lambda base, params: level_base_check(self, "WeisfeilerLehman", base, params, "label numbers",
                                                      "WL labels", "(n_iter + 1)"))
            self._initialized["base_graph_kernel"] = True
        if not self._initialized["n_iter"]:  # :111-115
            if type(self.n_iter) is not int or self.n_iter <= 0:
                raise TypeError("'n_iter' must be a positive integer")
            self._n_iter = self.n_iter + 1
            self._initialized["n_iter"] = True

    def _pack_for_base(self, X, len_ok):
        """One block per base kernel: the subtree kernel needs the adjacency structure only, the
        shortest-path base also the edge weights; the edge-histogram base never looks at the graph --
        its block has one "vertex" per edge-label entry and no edges, so that every WL round reproduces
        the same partition and K = (n_iter + 1) * K_EH, exactly what the reference computes by fitting
        one EdgeHistogram per level on unchanged edge labels (weisfeiler_lehman.py:157-169, 260-270)."""
        base = self._base_graph_kernel
        if isinstance(X, Block):  # packed input (datasets.read_tu)
            if base is EdgeHistogram:
                raise NotImplementedError("packed blocks carry no edge-label entries; pass the list of graphs")
            if base is SubgraphMatching:
                raise NotImplementedError("WeisfeilerLehman over SubgraphMatching needs every graph's edge dictionary "
                                          "and edge labels; pass the list of graphs")
            return X.require("wl")
        if base is EdgeHistogram:
            if not isinstance(X, Iterable):
                raise TypeError("input must be an iterable\n")
            X = list(X)
            pack(X, "wl", len_ok=len_ok)  # the reference builds the Graph + node labels first: same errors
            values = _edge_label_values(X)
            sizes = np.concatenate([[0], np.cumsum([len(v) for v in values])])
            return Block(sizes, np.zeros(int(sizes[-1]) + 1, dtype=np.int64), np.zeros(0, dtype=np.int64), None,
                         [l for v in values for l in v])
        if base is PyramidMatch and isinstance(X, Block):
            raise NotImplementedError("WeisfeilerLehman over PyramidMatch embeds every graph's adjacency matrix; pass "
                                      "the list of graphs")
        if base in (NeighborhoodSubgraphPairwiseDistance, OddSth) and isinstance(X, Block):
            raise NotImplementedError("WeisfeilerLehman over %s needs every graph's edge dictionary (edge labels, "
                                      "neighbour order); pass the list of graphs" % base.__name__)
        if base is ShortestPath:
            # the base kernel receives the edge DICTIONARY of every graph (weisfeiler_lehman.py:188, 218):
            # Dijkstra semantics whatever the input spelling; labels are the WL vertex set
            return pack(X, "wl", len_ok=len_ok, want_weights=True)
        return pack(X, "wl", len_ok=len_ok)

    def parse_input(self, X):
        if self._method_calling in (1, 2):
            if hasattr(self, "_X_diag"):
                delattr(self, "_X_diag")
            if not isinstance(X, (Iterable, Block)):
                raise TypeError("input must be an iterable\n")
            if self._base_graph_kernel in _WL_GRAPH_BASES and not isinstance(X, Block):
                X = list(X)
            block = self._pack_for_base(X, lambda n: n >= 2)  # weisfeiler_lehman.py:152
            self._nx = block.n_graphs
            ids, dictionary = label_ids(block.labels, None, sort_new=True)  # :199-206
            self._inv_labels = _LevelDictionaries(dictionary, self)
            fitted = Fitted(block, ids, dictionary)
            fitted.pm = self._pm_embed(X, block)
            fitted.base = self._base_data(X, block)
            self._fit_transformed = self._method_calling == 2
            return fitted
        if self._method_calling != 3:
            raise ValueError("method call must be called either from fit or fit-transform")
        if self._base_graph_kernel in _WL_GRAPH_BASES and not isinstance(X, Block):
            X = list(X)
        block = self._pack_for_base(X, lambda n: n in (2, 3))  # :367
        ids, _ = label_ids(block.labels, self._inv_labels[0], sort_new=True)  # :417-418
        fitted = Fitted(block, ids, self._inv_labels[0])
        fitted.pm = self._pm_embed(X, block)
        fitted.base = self._base_data(X, block)
        return fitted

    def _pm_embed(self, X, block):
        """PyramidMatch base: the embeddings of every level's fresh base kernel (weisfeiler_lehman.py:260-270,
        478-482), see pm_level_embeddings."""
        if self._base_graph_kernel is not PyramidMatch:
            return None
        d = self._params.get("d", 6)
        data, self.ms_host_embed_ = pm_level_embeddings(X, block, d, self._params.get("L", 4), self._n_iter,
                                                        "WeisfeilerLehman")
        return data

    def fit_transform(self, X, y=None):
        self._method_calling = 2
        self._is_transformed = False
        self.initialize()
        if X is None:
            raise ValueError("transform input cannot be None")
        self.X = self.parse_input(X)
        K, xdiag, _ = self._run(self.X, n_fit=self._nx)
        self._X_diag = xdiag
        return K

    def fit(self, X, y=None):
        self._is_transformed = False
        self._method_calling = 1
        self.initialize()
        if X is None:
            raise ValueError("`fit` input cannot be None")
        self.X = self.parse_input(X)
        return self

    def transform(self, X):
        self._method_calling = 3
        check_is_fitted(self, ["X", "_nx", "_inv_labels"])
        if X is None:
            raise ValueError("transform input cannot be None")
        if not isinstance(X, (Iterable, Block)):
            raise ValueError("input must be an iterable\n")
        Y = self.parse_input(X)
        if self._base_graph_kernel is OddSth and self.normalize and not getattr(self, "_fit_transformed", False):
            # the reference's diagonal() asks the fitted OddSth levels for self._phi_X, which they never set
            raise AttributeError("'OddSth' object has no attribute '_phi_X'")
        K, xdiag, ydiag = self._run(Fitted.concat(self.X, Y), n_fit=self._nx)
        self._X_diag = xdiag
        self._Y_diag = ydiag
        self._is_transformed = True
        return K

    def _device_features(self, eng):
        if self._base_graph_kernel is ShortestPath:
            return eng.wl_sp_features(self._n_iter - 1, dijkstra_order=True)  # the base kernel gets edge dictionaries
        return eng.wl_features(self._n_iter - 1)

    def diagonal(self):
        check_is_fitted(self, ["X"])
        if self._base_graph_kernel is OddSth and not getattr(self, "_fit_transformed", False):
            if not getattr(self, "_is_transformed", False):
                raise NotFittedError("This OddSth instance is not fitted yet. Call 'fit' with appropriate arguments "
                                     "before using this estimator.")
            raise AttributeError("'OddSth' object has no attribute '_phi_X'")
        try:
            check_is_fitted(self, ["_X_diag"])
        except NotFittedError:
            _, self._X_diag, _ = self._run(self.X, n_fit=self._nx, want_matrix=False)
        if getattr(self, "_is_transformed", False):
            return self._X_diag, self._Y_diag
        return self._X_diag

    def _base_data(self, X, block):
        """NeighborhoodSubgraphPairwiseDistance / OddSth / SubgraphMatching base: see base_graph_data."""
        base = self._base_graph_kernel
        if base not in _WL_GRAPH_BASES or base is PyramidMatch:
            return None
        return base_graph_data(X, block, base, getattr(self, "_sm", None), "WeisfeilerLehman")

    def _relabel(self, eng, block, ids):
        """Pack the WL vertex set and relabel it on the device: every level's classes stay on `eng` (gk_wl_features)."""
        eng.pack(block.graph_ptr, block.row_ptr, block.col_idx, ids, None, None)
        eng.wl_features(self._n_iter - 1)

    def _level_classes(self, eng, block, ids):
        """[V, n_iter + 1]: the WL class of every packed vertex at every level, level 0 its label id (gk_wl_labels)."""
        self._relabel(eng, block, ids)
        return np.stack([ids] + [eng.wl_labels(lv, block.n_vertices) for lv in range(1, self._n_iter)], axis=1)

    def _base_run(self, data, n_fit, want_matrix=True, row_range=None, device_ptr=None):
        """WL over PyramidMatch, NeighborhoodSubgraphPairwiseDistance, OddSth or SubgraphMatching: K = sum over the levels
        of the base kernel on the level's labels (weisfeiler_lehman.py:260-270), by that base's level route.  NSPD and
        OddSth read the reference's label numbers, so the device partition is numbered on the host first."""
        base, p = self._base_graph_kernel, self._params
        block, ids = data.block, data.ids
        if base is PyramidMatch:
            relabel = functools.partial(self._relabel, block=block, ids=ids) if p.get("with_labels", True) else None
            return pm_level_run(self, data.pm, block, relabel, self._n_iter, p.get("L", 4), p.get("d", 6), n_fit,
                                want_matrix, row_range, device_ptr)
        classes = None
        if not (base is SubgraphMatching and self._sm.kv is None):
            with _lib.engine(getattr(self, "device_", None)) as eng:
                classes = self._level_classes(eng, block, ids)
        if base is SubgraphMatching:
            return sm_level_run(self, data.base, classes, True, self._n_iter - 1, n_fit, want_matrix, row_range,
                                device_ptr)
        t0 = time.perf_counter()
        _, labels = wl_reference_dictionaries(np.asarray(block.row_ptr), np.asarray(block.col_idx), ids,
                                              len(self.X.dictionary), classes.T,
                                              n_fit_vertices=int(np.asarray(block.graph_ptr)[n_fit]))
        self.ms_host_numbering_ = (time.perf_counter() - t0) * 1e3
        if base is OddSth:
            return self._wl_odd_run(data.base, labels, n_fit, want_matrix, row_range)
        return self._wl_nspd_run(data.base, labels, n_fit, want_matrix, row_range)

    def _wl_odd_run(self, data, labels, n_fit, want_matrix, row_range):
        b = data.block
        ids, rank, off = [], [], 0
        for lab in labels:
            L = np.asarray(lab, dtype=np.int64)[data.src]
            if len(L) and L.max() >= 2 ** 31:
                raise NotImplementedError("WeisfeilerLehman over OddSth: a WL label of 2^31 or more")
            uniq, inv = np.unique(L, return_inverse=True)
            ids.append(inv.reshape(-1) + off)  # str(label) identities: one id per label, disjoint across levels
            rank.append(L)                      # Kahn's order compares the label values themselves
            off += len(uniq)
        if off >= 2 ** 31:
            raise NotImplementedError("WeisfeilerLehman over OddSth: 2^31 or more labels over all levels")
        h = self._params.get("h")
        with _lib.engine(getattr(self, "device_", None)) as eng:
            eng.pack(b.graph_ptr, b.row_ptr, b.col_idx, ids[0], None, None)
            self.stats_ = eng.wl_odd_features(-1 if h is None else h, self._n_iter - 1, np.stack(ids), np.stack(rank))
            K, xd, yd = eng.gram(b.n_graphs, n_fit=n_fit, normalize=bool(self.normalize) and want_matrix,
                                 nan_to_num=True, out=None if want_matrix else False, row_range=row_range,
                                 stats=self.stats_)
        if self.verbose:
            print(type(self).__name__, self.stats_.as_dict())
        return K, xd, yd

    def _wl_nspd_run(self, data, labels, n_fit, want_matrix, row_range):
        def levels():
            for lab in labels:
                uniq, inv = np.unique(np.asarray(lab, dtype=np.int64)[data.src], return_inverse=True)
                yield inv.reshape(-1), [str(int(u)) for u in uniq]
        p = self._params
        return nspd_level_sum(self, data, levels(), self._n_iter, n_fit, want_matrix, row_range, p.get("r", 3),
                              p.get("d", 4))

    def _run(self, data, n_fit, want_matrix=True):
        """`data`: a Fitted, the fitted graphs first.  The plain subtree fit_transform (square, un-normalised) is ONE C
        call, gk_wl_gram: relabel, column statistics, head/tail decision on the device, GEMM, tail and delivery with a
        single host synchronisation."""
        block, ids = data.block, data.ids
        if self._base_graph_kernel in _WL_GRAPH_BASES:
            return self._base_run(data, n_fit, want_matrix)
        if (want_matrix and not self.normalize and n_fit == block.n_graphs and self._base_graph_kernel is VertexHistogram
                and type(self) is WeisfeilerLehman):
            with _lib.engine(getattr(self, "device_", None)) as eng:
                eng.pack(block.graph_ptr, block.row_ptr, block.col_idx, ids, block.weights, block.attrs)
                K, xd, self.stats_ = eng.wl_gram(self._n_iter - 1, want_diag=True)
            if self.verbose:
                print(type(self).__name__, self.stats_.as_dict())
            return K, xd, None
        return super()._run(block, ids, n_fit, want_matrix)

    def _export_level_dictionaries(self):
        """`_inv_labels[i]` for i >= 1 (weisfeiler_lehman.py:257): the fitted graphs are relabelled on the device, the
        per-level classes come back through `gk_wl_labels`, and the host names every class the way the reference
        does.  Also keeps `wl_labels_`: the reference's compressed label of every packed vertex, per level."""
        check_is_fitted(self, ["X", "_nx"])
        block, ids = self.X.block, self.X.ids
        with _lib.engine(getattr(self, "device_", None)) as eng:
            classes = self._level_classes(eng, block, ids)
        out, self.wl_labels_ = wl_reference_dictionaries(np.asarray(block.row_ptr), np.asarray(block.col_idx), ids,
                                                         len(self.X.dictionary), classes.T)
        return out


def nspd_level_sum(est, data, levels, n_levels, n_fit, want_matrix, row_range, r, d):
    """NeighborhoodSubgraphPairwiseDistance under a relabelling framework (estimator `est`): `levels` yields, level
    by level, the label id of every base vertex and the label string of every id; each level packs its labels and
    tokens, runs gk_nspd_features, and gk_wl_level_sum adds its un-normalised K into a device-resident sum in level
    order.  Normalised as the frameworks do: by the sum's diagonal after fit_transform, by the base diagonals (the
    number of (radius, distance) levels, per level) after a transform.  Returns (K, xdiag, ydiag)."""
    graphs = data.graphs
    if r > 0 and max(g[0] for g in graphs) >= 65535:  # the device refuses it too; do not pack it first
        raise NotImplementedError("NeighborhoodSubgraphPairwiseDistance: r > 0 with a graph of 65535 or more "
                                  "vertices")
    nsp = NeighborhoodSubgraphPairwiseDistance(r=r, d=d)
    gp, rp, ci, _, el, sh, tok0 = nsp._pack([(n, e, ["0"] * n, l) for n, e, _, l in graphs])
    elabels = [tok0.el_bytes[tok0.el_off[i]:tok0.el_off[i + 1]].tobytes().decode("utf-8")
               for i in range(tok0.n_elabels)]
    N = len(gp) - 1
    square = n_fit == N
    rows_total = N if square else N - n_fit
    rb, re_ = (0, rows_total) if row_range is None else row_range
    with _lib.engine(getattr(est, "device_", None)) as eng:
        for lv, (ids, strings) in enumerate(levels):
            tokens = _NspdTokens(d, strings, elabels)
            eng.pack(gp, rp, ci, ids, None, None)
            est.stats_, mask = eng.nspd_features(r, d, sh, el, tokens)
            if want_matrix:
                eng.wl_level_sum(lv, n_fit, (rb, re_))
        # diagonal() of every fitted level: its number of (radius, distance) levels (the reference's constant)
        def n_rd(m):
            top = max((int(x).bit_length() for x in m), default=0)
            return (r + 1) * top
        xd_lv = np.full(n_fit, float(n_rd(mask[:n_fit])))
        yd_lv = None if square else np.full(N - n_fit, float(n_rd(mask[n_fit:])))
        xd_sum = xd_lv.copy()
        yd_sum = None if yd_lv is None else yd_lv.copy()
        for _ in range(1, n_levels):
            xd_sum += xd_lv
            if yd_sum is not None:
                yd_sum += yd_lv
        if not want_matrix:
            return None, xd_sum, yd_sum
        if square:
            full = rb == 0 and re_ == N
            K, kd = eng.wl_level_sum_fetch(re_ - rb, n_fit, normalize=bool(est.normalize), want_kdiag=full)
            return K, kd, None
        xd = getattr(est, "_X_diag", None)
        xd = xd_sum if xd is None else np.asarray(xd, dtype=np.float64).reshape(-1)
        K, _ = eng.wl_level_sum_fetch(re_ - rb, n_fit, normalize=bool(est.normalize), xdiag=xd, ydiag=yd_sum)
        return K, xd, yd_sum


def sm_level_features(eng, sm, data, classes, refine, n_iter):
    """SubgraphMatching `sm` under a relabelling framework, set up on `eng` for one enumeration of every level:
    `data` (_WlBaseData) the base graphs, `classes` [V, n_levels] the class of every packed framework vertex per level
    (None with kv=None: every level is level 0).  Levels that refine each other (WL's) run gk_sm_wl_features, others
    (HadamardCode's) gk_sm_hc_features; `n_iter` is the framework's own.  Returns the stats."""
    level_ids = None if classes is None else classes[data.src]
    graphs, v0 = [], 0
    for n, edges, _, el in data.graphs:
        graphs.append((n, edges, None if level_ids is None else level_ids[v0:v0 + n, 0].tolist(), el))
        v0 += n
    gp, rp, ci, lab, elids, _, et, flags = sm._pack(graphs)
    eng.pack(gp, rp, ci, lab, None, None)
    features = eng.sm_wl_features if refine else eng.sm_hc_features
    return features(int(sm.k), n_iter, level_ids, sm.lambdas_, et, elids, flags)


def sm_level_run(est, data, classes, refine, n_iter, n_fit, want_matrix, row_range=None, device_ptr=None):
    """SubgraphMatching (est._sm) under a relabelling framework `est`: K = sum over the levels of SubgraphMatching on
    the level's classes, from one clique enumeration per pair (DESIGN 4.23, 4.24); see sm_level_features.
    Returns (K, xdiag, ydiag)."""
    with _lib.engine(getattr(est, "device_", None)) as eng:
        est.stats_ = sm_level_features(eng, est._sm, data, classes, refine, n_iter)
        K, xd, yd = eng.gram(len(data.graphs), n_fit=n_fit, normalize=bool(est.normalize) and want_matrix,
                             nan_to_num=True, out=None if want_matrix else False, row_range=row_range,
                             device_ptr=device_ptr, stats=est.stats_)
    if est.verbose:
        print(type(est).__name__, est.stats_.as_dict())
    return K, xd, yd


def pm_level_run(est, pm, block, relabel, n_levels, L, d, n_fit, want_matrix, row_range=None, device_ptr=None):
    """PyramidMatch under a relabelling framework `est`: every level's classes label a PyramidMatch of its own over
    the level's embeddings `pm` (_PmData, see pm_level_embeddings).  `relabel(eng)` packs `block` and relabels it on
    the device, where gk_pm_features reads every level's classes; None (with_labels=False): no labels, no relabelling.
    Returns (K, xdiag, ydiag)."""
    with _lib.engine(getattr(est, "device_", None)) as eng:
        if relabel is None:
            eng.pack(block.graph_ptr, block.row_ptr, block.col_idx, None, None, None)
        else:
            relabel(eng)
        est.stats_ = eng.pm_features(L, d, pm.U, pm.n_cols, n_iter=n_levels - 1,
                                     flags=0 if relabel is None else _lib.GK_PM_WL_LABELS, skip=pm.skip)
        K, xd, yd = eng.gram(block.n_graphs, n_fit=n_fit, normalize=bool(est.normalize) and want_matrix,
                             nan_to_num=True, out=None if want_matrix else False, row_range=row_range,
                             device_ptr=device_ptr, stats=est.stats_)
    if est.verbose:
        print(type(est).__name__, est.stats_.as_dict())
    return K, xd, yd


def base_graph_data(X, block, base, sm, who):
    """NeighborhoodSubgraphPairwiseDistance / OddSth / SubgraphMatching under a relabelling framework (`sm`: the
    SubgraphMatching that checks the elements): every element's graph as that base kernel packs it, and `src`, the
    packed vertex of every base vertex (the base kernel sees the level labels through the element's labels dictionary,
    whose key order is the packed block's)."""
    gp = np.asarray(block.graph_ptr, dtype=np.int64)
    src, graphs, els = [], [], []
    for x in X:
        from_graph = isinstance(x, Graph)
        if from_graph:
            x = x.as_element()
        x = list(x)
        if len(x) == 0:
            continue
        loc = {k: i for i, k in enumerate(x[1].keys())}
        if base is NeighborhoodSubgraphPairwiseDistance:
            if len(x) != 3:  # the element the reference hands on is (edges, labels) + edge labels
                raise TypeError(_NSPD_ELEMENT_MSG)
            n, edges, _, el, order = _nspd_graph(x[0], x[1], x[2], with_order=True)
            graphs.append((n, edges, None, el))
        elif base is SubgraphMatching:
            # the reference hands on (edges, labels) + extras, extras starting with the edge labels when the
            # element has them (weisfeiler_lehman.py:157-176): without them SubgraphMatching gets two entries
            if len(x) != 3 or (from_graph and not x[2]):
                raise TypeError(_SM_ELEMENT_MSG)
            n, edges, _, el = sm._graph(x[0], None, x[2] if x[2] else None, need_v=False)
            order = adjacency_and_order(x[0])[1]
            graphs.append((n, edges, None, el))
        else:
            if type(x[0]) is dict and x[0] and all(type(d) is list for d in x[0].values()) and not all(x[0].values()):
                raise ValueError("vertex not inside edge dictionary")
            els.append([x[0], x[1]])
            order = adjacency_and_order(x[0])[1]
        src.append([loc.get(k, -1) for k in order])
    out = _WlBaseData()
    cols = []
    for g, rows in enumerate(src):
        rows = np.asarray(rows, dtype=np.int64)
        if np.any(rows < 0):
            raise NotImplementedError("%s over %s: a vertex of a graph's edges has no label" % (who, base.__name__))
        cols.append(rows + gp[g])
    out.src = np.concatenate(cols) if cols else np.zeros(0, dtype=np.int64)
    out.wl_vertices = int(gp[-1])
    if base in (NeighborhoodSubgraphPairwiseDistance, SubgraphMatching):
        out.graphs = graphs
    else:
        b = pack(els, "sp", need_labels=True, len_ok=lambda n: n == 2, type_error_msg=_ODD_ELEMENT_MSG,
                 keep_edge_order=True)
        if b.n_vertices != len(out.src):
            raise NotImplementedError(who + " over OddSth: a graph's vertices are not those of its edges")
        out.block = b
    return out


def pm_level_embeddings(X, block, d, L, n_sets, who):
    """PyramidMatch under a relabelling framework: the embeddings of every level's fresh base kernel, n_sets passes
    over the graphs, level-major, each one eigs / eig call per graph.  The base kernel sees every graph's adjacency:
    its vertices are those of the element's adjacency matrix (range(n), or the sorted symbols of the edge dictionary),
    each with its own label.  The packed block lists a graph's vertices in the order of its labels dictionary and also
    holds labelled vertices outside the edge dictionary; so every embedding row is moved to its vertex's packed
    position, and the vertices the base kernel does not see are skipped (they never change another vertex's label).
    Returns (_PmData, host embedding milliseconds)."""
    from .packing import adjacency_and_order
    import time
    mats, src = [], []
    n_pm = 0
    for x in X:
        if isinstance(x, Graph):
            x = x.as_element()
        x = list(x)
        if len(x) == 0:
            continue
        A, order = adjacency_and_order(x[0])
        loc = {k: i for i, k in enumerate(order)}
        rows = [loc.get(k, -1) for k in x[1].keys()]  # the packed vertices, in the pack's order
        if sum(r >= 0 for r in rows) != len(order):
            raise NotImplementedError(who + " over PyramidMatch: a vertex of a graph's edge dictionary has no label")
        src.extend(r + n_pm if r >= 0 else -1 for r in rows)
        mats.append(A)
        n_pm += A.shape[0]
    src = np.asarray(src, dtype=np.int64)
    if len(src) != block.n_vertices:
        raise NotImplementedError(who + " over PyramidMatch: the packed vertices are not the labelled ones")
    t0 = time.perf_counter()
    U_pm, n_cols = pm_embed_sets(mats, d, n_sets)
    ms = (time.perf_counter() - t0) * 1e3
    pm_check_cells(U_pm, n_cols, np.array([A.shape[0] for A in mats]), L)
    seen = src >= 0
    U = np.zeros((n_sets, len(src), d))
    U[:, seen] = U_pm[:, src[seen]]
    return _PmData(np.diff(np.asarray(block.graph_ptr)), U, n_cols, None, skip=None if seen.all() else ~seen), ms


class _WlBaseData:
    """What WL over NeighborhoodSubgraphPairwiseDistance / OddSth keeps per call: the base kernel's graphs (NSPD: (n,
    edges, -, edge label strings); OddSth: its packed block) and `src`, the WL vertex of every base vertex."""

    graphs = None
    block = None

    @staticmethod
    def concat(a, b):
        out = _WlBaseData()
        out.src = np.concatenate([a.src, b.src + a.wl_vertices])
        out.wl_vertices = a.wl_vertices + b.wl_vertices
        if a.graphs is not None:
            out.graphs = a.graphs + b.graphs
        else:
            out.block = Block.concat(a.block, b.block)
        return out


# ------------------------------------------------------------------------------
class WeisfeilerLehmanOptimalAssignment(Kernel):
    """Weisfeiler-Lehman optimal-assignment kernel (weisfeiler_lehman_optimal_assignment.py:19-481):
    K[i, j] = sum over the WL label hierarchy of min(#vertices of i, #vertices of j) carrying the label.

    The reference fills K with an O(N^2) Python loop of histogram intersections (:257-266); here the WL
    feature block is expanded to unary form on the device (`gk_wl_oa_features`) and the same Gram as the
    subtree kernel returns the intersections exactly.  `sparse` only selects the reference's storage
    of Hs and does not change K; it is accepted and ignored."""

    _graph_format = "dictionary"
    _nan_to_num = True

    def __init__(self, n_jobs=None, verbose=False, normalize=False, n_iter=5, sparse=False):
        super().__init__(n_jobs=n_jobs, verbose=verbose, normalize=normalize)
        self.n_iter = n_iter
        self.sparse = sparse
        self._initialized.update({"n_iter": False, "sparse": True})

    def initialize(self):
        super().initialize()
        if not self._initialized["n_iter"]:  # :68-72
            if type(self.n_iter) is not int or self.n_iter <= 0:
                raise TypeError("'n_iter' must be a positive integer")
            self._n_iter = self.n_iter + 1
            self._initialized["n_iter"] = True
        if not self._initialized["sparse"]:
            self._initialized["sparse"] = False

    def parse_input(self, X):
        msg = ("each element of X must be either a graph object or a list with at least a graph like object and "
               "node labels dict \n")
        if self._method_calling in (1, 2):
            if hasattr(self, "_X_diag"):
                delattr(self, "_X_diag")
            if isinstance(X, Block):  # packed input (datasets.read_tu)
                block = X.require("sp", "wloa", "core")
            elif not isinstance(X, Iterable):
                raise TypeError("input must be an iterable\n")
            else:
                block = pack(X, "wloa", len_ok=lambda n: n >= 2, type_error_msg=msg)  # :113
            self._nx = block.n_graphs
            ids, dictionary = label_ids(block.labels, None, sort_new=True)  # :157-161
            self._inv_labels = {0: dictionary}
            self._hierarchy = {"root": {"parent": None, "w": 0, "omega": 0}}  # fitted marker; the tree lives on the device
            return Fitted(block, ids, dictionary)
        if self._method_calling != 3:
            raise ValueError("method call must be called either from fit or fit-transform")
        if isinstance(X, Block):
            block = X.require("sp", "wloa", "core")
        else:
            try:
                block = pack(X, "wloa", len_ok=lambda n: n in (2, 3), type_error_msg=msg)  # :323
            except TypeError as e:  # transform raises ValueError for malformed elements (:344-346)
                raise ValueError("each element of X must have at least one and at most 3 elements\n") from e
        ids, _ = label_ids(block.labels, self._inv_labels[0], sort_new=True)  # :356-359
        return Fitted(block, ids, self._inv_labels[0])

    def fit_transform(self, X, y=None):
        self._method_calling = 2
        self._is_transformed = False
        self.initialize()
        if X is None:
            raise ValueError("transform input cannot be None")
        self.X = self.parse_input(X)
        K, xdiag, _ = self._run(self.X.block, self.X.ids, n_fit=self._nx)
        self._X_diag = xdiag
        return K

    def transform(self, X):
        self._method_calling = 3
        check_is_fitted(self, ["X", "_nx", "_hierarchy", "_inv_labels"])
        if X is None:
            raise ValueError("transform input cannot be None")
        if not isinstance(X, (Iterable, Block)):
            raise ValueError("input must be an iterable\n")
        Y = self.parse_input(X)
        K, xdiag, ydiag = self._run(Block.concat(self.X.block, Y.block), np.concatenate([self.X.ids, Y.ids]),
                                    n_fit=self._nx)
        self._X_diag = xdiag
        self._Y_diag = ydiag
        self._is_transformed = True
        return K

    def _device_features(self, eng):
        return eng.wl_oa_features(self._n_iter - 1)


# ------------------------------------------------------------------------------
class ShortestPath(Kernel):
    """Shortest-path kernel (shortest_path.py:167-515): features are
    (l(u), l(v), d(u,v)) triples (or d(u,v) alone with with_labels=False) over ordered
    vertex pairs at finite distance; K = Phi Phi^T."""

    def __init__(self, n_jobs=None, normalize=False, verbose=False, with_labels=True, algorithm_type="auto"):
        super().__init__(n_jobs=n_jobs, normalize=normalize, verbose=verbose)
        self.with_labels = with_labels
        self.algorithm_type = algorithm_type
        self._initialized.update({"with_labels": False, "algorithm_type": False})

    def initialize(self):
        if not self._initialized["n_jobs"]:  # shortest_path.py:239-242
            if self.n_jobs is not None:
                warnings.warn("no implemented parallelization for ShortestPath")
            self._initialized["n_jobs"] = True
        if not self._initialized["algorithm_type"]:  # :244-252
            if self.algorithm_type == "auto":
                self._graph_format = "auto"
            elif self.algorithm_type == "floyd_warshall":
                self._graph_format = "adjacency"
            elif self.algorithm_type == "dijkstra":
                self._graph_format = "dictionary"
            else:
                raise ValueError('Unsupported "algorithm_type"')
        self._lt = "vertex" if self.with_labels else "none"

    def parse_input(self, X):
        wl = bool(self.with_labels)
        # Floyd-Warshall treats a 0 entry as "no edge" (graph.py:1786); Dijkstra walks every
        # listed edge.  "auto" picks FW for adjacency input and Dijkstra for dictionaries, so
        # zero-weight dictionary edges only disappear when FW is forced.
        if isinstance(X, Block):  # packed input (datasets.read_tu): unit weights, dictionary semantics
            block = X.require("sp", labels=wl)
        else:
            block = pack(X, "sp", need_labels=wl, len_ok=lambda n: n in (2, 3) or (n == 1 and not wl),
                         want_weights=True, fw_zero_is_absent=self.algorithm_type == "floyd_warshall",
                         type_error_msg="each element of X must have at least one and at most 3 elements\n")
        # real-valued weights: feature keys compare path lengths by exact float equality (shortest_path.py:472, 511)
        # and the reference's Dijkstra and Floyd-Warshall round differently; the device reproduces whichever the
        # reference would run (k-ordered fp64 Floyd-Warshall, or the Dijkstra-order fixed point of sp_dijkstra_order_apsp)
        dj = _path_sum_order(block, self.algorithm_type)
        if self._method_calling in (1, 2):
            self._dijkstra_order = dj
        elif dj != getattr(self, "_dijkstra_order", dj) and block.weights is not None:
            self._dijkstra_order = self._dijkstra_order or dj
        if self._method_calling in (1, 2):
            self._nx = block.n_graphs
            if wl:
                ids, dictionary = label_ids(block.labels, None, sort_new=False)
            else:
                ids, dictionary = None, {}
            self._enum = dictionary  # fitted marker (the reference keeps the feature enumeration here)
            return Fitted(block, ids, dictionary)
        self._ny = block.n_graphs
        if wl:
            ids, _ = label_ids(block.labels, self.X.dictionary, sort_new=False)
        else:
            ids = None
        return Fitted(block, ids, self.X.dictionary)

    def fit_transform(self, X, y=None):
        self._method_calling = 2
        self.fit(X)  # resets _method_calling to 1 like shortest_path.py:392-393
        K, xdiag, _ = self._run(self.X.block, self.X.ids, n_fit=self._nx)
        self._X_diag = xdiag
        return K

    def transform(self, X):
        self._method_calling = 3
        check_is_fitted(self, ["X", "_nx", "_enum"])
        if X is None:
            raise ValueError("transform input cannot be None")
        Y = self.parse_input(X)
        ids = None if self.X.ids is None else np.concatenate([self.X.ids, Y.ids])
        K, xdiag, ydiag = self._run(Block.concat(self.X.block, Y.block), ids, n_fit=self._nx)
        self._X_diag = xdiag
        self._Y_diag = ydiag
        self._is_transformed = True
        return K

    def diagonal(self):
        out = super().diagonal()
        if isinstance(out, tuple):  # shortest_path.py:359-366: X diagonal as a column
            return np.reshape(out[0], (-1, 1)), out[1]
        return np.reshape(out, (-1, 1))

    def _device_features(self, eng):
        return eng.sp_features(with_labels=bool(self.with_labels), dijkstra_order=bool(getattr(self, "_dijkstra_order", False)))


class ShortestPathAttr(Kernel):
    """Shortest-path kernel on node attributes (shortest_path.py:16-164)."""

    def __init__(self, n_jobs=None, normalize=False, verbose=False, algorithm_type="auto", metric=np.dot):
        super().__init__(n_jobs=n_jobs, normalize=normalize, verbose=verbose)
        self.algorithm_type = algorithm_type
        self.metric = metric
        self._initialized.update({"algorithm_type": False, "metric": False})

    def initialize(self):
        super().initialize()
        if not self._initialized["algorithm_type"]:
            if self.algorithm_type not in ("auto", "floyd_warshall", "dijkstra"):
                raise ValueError("Unsupported value " + str(self.algorithm_type) + ' for "algorithm_type"')
            self._initialized["algorithm_type"] = True
        if not self._initialized["metric"]:
            if not callable(self.metric):
                raise TypeError('"metric" must be callable')
            self._initialized["metric"] = True

    def _bilinear(self):
        """The explicit feature map (and with it the tensor-core Gram) is valid for the default metric only."""
        return self.metric is np.dot

    def parse_input(self, X):
        if not self._bilinear():
            return self._parse_pairs(X)
        if isinstance(X, Block):  # packed input (datasets.read_tu(prefer_attr_nodes=True))
            if X.require("sp", labels=False).attrs is None:
                raise ValueError("Graph does not have any labels for vertices.")
            return Fitted(X, None, {})
        block = pack(X, "sp", need_labels=True, len_ok=lambda n: n in (2, 3), want_weights=True,
                     fw_zero_is_absent=self.algorithm_type == "floyd_warshall", attributes=True,
                     type_error_msg="each element of X must be either a graph or an iterable with at least 2 and at "
                                    "most 3 elements\n")
        self._dijkstra_order = _path_sum_order(block, self.algorithm_type) or getattr(self, "_dijkstra_order", False)
        return Fitted(block, None, {})

    # ---- a user metric: shortest-path matrices on the device, the reference's per-pair contraction on the host
    def _parse_pairs(self, X):
        """shortest_path.py:77-129 for a callable metric: one (S, phi) tuple per graph.  S comes from the device APSP
        kernels (gk_spattr_features -> gk_sp_distances; the path-sum order the reference would use), phi are the
        attribute rows.  The metric is a Python callback per attribute pair by definition, so the contraction of
        shortest_path.py:130-164 runs on the host (`pairwise_operation`), through the generic driver of the base
        class (kernel.py:236-296)."""
        if isinstance(X, Block):
            block = X.require("sp", labels=False)
            if block.attrs is None:
                raise ValueError("Graph does not have any labels for vertices.")
        else:
            block = pack(X, "sp", need_labels=True, len_ok=lambda n: n in (2, 3), want_weights=True,
                         fw_zero_is_absent=self.algorithm_type == "floyd_warshall", attributes=True,
                         type_error_msg="each element of X must be either a graph or an iterable with at least 2 and at "
                                        "most 3 elements\n")
        dj = _path_sum_order(block, self.algorithm_type)
        items = []
        with _lib.engine(getattr(self, "device_", None)) as eng:
            eng.pack(block.graph_ptr, block.row_ptr, block.col_idx, None, block.weights, block.attrs)
            self.stats_ = eng.spattr_features(dijkstra_order=bool(dj))
            gp = block.graph_ptr
            for g in range(block.n_graphs):
                n = int(gp[g + 1] - gp[g])
                S = eng.sp_distances(g, n) if n else np.zeros((0, 0))
                items.append((S, np.array(block.attrs[gp[g]:gp[g + 1]], dtype=float)))
        return items

    def pairwise_operation(self, x, y):
        """shortest_path.py:130-164, vectorised over the path lengths: sum over ordered vertex pairs (i, j) of x and
        (k, m) of y with equal finite shortest-path length of metric(phi_x[i], phi_y[k]) * metric(phi_x[j], phi_y[m])."""
        Sx, phi_x = x
        Sy, phi_y = y
        nx, ny = Sx.shape[0], Sy.shape[0]
        if nx < 2 or ny < 2:
            return 0
        M = np.empty((nx, ny), dtype=float)
        for i in range(nx):
            for k in range(ny):
                M[i, k] = self.metric(phi_x[i], phi_y[k])
        offx, offy = ~np.eye(nx, dtype=bool), ~np.eye(ny, dtype=bool)
        fx, fy = offx & np.isfinite(Sx), offy & np.isfinite(Sy)
        kernel = 0.0
        for d in np.intersect1d(np.unique(Sx[fx]), np.unique(Sy[fy])):
            Ax = (fx & (Sx == d)).astype(float)
            Ay = fy & (Sy == d)
            kernel += float(np.sum((M.T @ Ax @ M)[Ay]))
        return kernel

    def diagonal(self):
        if not self._bilinear():
            return self._pairwise_diagonal()
        return super().diagonal()

    def fit_transform(self, X, y=None):
        self.initialize()
        if not self._bilinear():
            return self._pairwise_fit_transform(X)
        self._method_calling = 2
        self.fit(X)
        K, xdiag, _ = self._run(self.X.block, None, n_fit=self.X.block.n_graphs)
        self._X_diag = xdiag
        if self.normalize:
            self._warn_unnormalizable(xdiag)
        return K

    def transform(self, X):
        if not self._bilinear():
            return self._pairwise_transform(X)
        self._method_calling = 3
        check_is_fitted(self, ["X"])
        if X is None:
            raise ValueError("`transform` input cannot be None")
        Y = self.parse_input(X)
        K, xdiag, ydiag = self._run(Block.concat(self.X.block, Y.block), None, n_fit=self.X.block.n_graphs)
        self._X_diag = xdiag
        self._Y_diag = ydiag
        self._is_transformed = True
        if self.normalize:
            self._warn_unnormalizable(xdiag, ydiag)
        return K

    def _device_features(self, eng):
        return eng.spattr_features(dijkstra_order=bool(getattr(self, "_dijkstra_order", False)))


# ------------------------------------------------------------------------------
# GraphHopper node kernels on (M, attributes[, squared norms]) tuples (graph_hopper.py:295-365).  Module-level
# functions, so that a fitted estimator pickles; the device computes the same values without these callbacks.
def gh_linear_kernel(x, y):
    """sum of <M_v, M_v'> <x_v, x_v'> over node pairs (graph_hopper.py:295-313)."""
    M_i, NA_i = x[:2]
    M_j, NA_j = y[:2]
    return float(np.dot(np.dot(M_i, M_j.T).flat, np.dot(NA_i, NA_j.T).flat))


def gh_gaussian_kernel(x, y, mu=1.0):
    """sum of <M_v, M_v'> exp(-mu ||x_v - x_v'||^2) over node pairs (graph_hopper.py:316-339)."""
    M_i, NA_i = x[:2]
    M_j, NA_j = y[:2]
    sq = np.sum((NA_i[:, None, :] - NA_j[None, :, :]) ** 2, axis=2)
    return float(np.dot(np.dot(M_i, M_j.T).flat, np.exp(-mu * sq).flat))


def gh_bridge_kernel(x, y):
    """sum of <M_v, M_v'> max(0, (4 - ||x_v - x_v'||) / 4) over node pairs (graph_hopper.py:342-365)."""
    M_i, NA_i = x[:2]
    M_j, NA_j = y[:2]
    dist = np.sqrt(np.sum((NA_i[:, None, :] - NA_j[None, :, :]) ** 2, axis=2))
    return float(np.dot(np.dot(M_i, M_j.T).flat, np.maximum(0.0, (4.0 - dist) / 4.0).flat))


class GraphHopper(Kernel):
    """GraphHopper kernel (graph_hopper.py:19-449): K(G, G') = sum over vertex pairs of <M_v, M_v'> k(x_v, x_v'),
    where M_v counts the shortest paths through v by the position of v on the path and the path length.

    `kernel_type` is "linear", "gaussian" (mu = 1), ("gaussian", mu), "bridge" or a callable on the reference's
    (M reshaped to n x m^2, attributes) tuples.  The node maps are built on the device for every kernel type; the
    three named node kernels also run their Gram there, a callable is contracted pair by pair on the host.  Only
    unit edge weights are supported (the shortest-path DAG of the reference is defined for unweighted graphs)."""

    _graph_format = "all"

    def __init__(self, n_jobs=None, normalize=False, verbose=False, kernel_type="linear"):
        super().__init__(n_jobs=n_jobs, normalize=normalize, verbose=verbose)
        self.kernel_type = kernel_type
        self._initialized.update({"kernel_type": False})

    def initialize(self):
        super().initialize()
        if not self._initialized["kernel_type"]:  # graph_hopper.py:51-85
            kt = self.kernel_type
            if type(kt) is str:
                if kt == "linear":
                    self.metric_, self.calculate_norm_, self._node_kernel = gh_linear_kernel, False, (_lib.GK_GH_LINEAR, 1.0)
                elif kt == "gaussian":
                    self.metric_ = functools.partial(gh_gaussian_kernel, mu=1.0)
                    self.calculate_norm_, self._node_kernel = True, (_lib.GK_GH_GAUSSIAN, 1.0)
                elif kt == "bridge":
                    self.metric_, self.calculate_norm_, self._node_kernel = gh_bridge_kernel, False, (_lib.GK_GH_BRIDGE, 1.0)
                else:
                    raise ValueError('Unsupported kernel with name "' + str(kt) + '"')
            elif type(kt) is tuple and len(kt) == 2 and kt[0] == "gaussian" and isinstance(kt[1], Real):
                self.metric_ = functools.partial(gh_gaussian_kernel, mu=float(kt[1]))
                self.calculate_norm_, self._node_kernel = True, (_lib.GK_GH_GAUSSIAN, float(kt[1]))
            elif callable(kt):
                self.metric_, self.calculate_norm_, self._node_kernel = kt, False, None
            else:
                raise TypeError('Unrecognized "kernel_type": can either be a str from the supported: "linear", '
                                '"gaussian", "bridge" or tuple ("gaussian", mu) or a callable.')
            self._initialized["kernel_type"] = True

    # ---- input
    def _pack(self, X):
        """Packed block of X: adjacency semantics (entries > 0 are edges, self-loops take no part), node attributes
        as vectors, the reference's element and attribute errors (graph_hopper.py:106-164)."""
        if isinstance(X, Block):  # datasets.read_tu(prefer_attr_nodes=True)
            block = X.require("sp", labels=False)
            if block.attrs is None:
                raise ValueError("Graph does not have any labels for vertices.")
        else:
            if not isinstance(X, Iterable):
                raise TypeError("input must be an iterable\n")
            X = list(X)
            msg = "each element of X must be either a graph object or a list with at least a graph like object and node, "
            from .packing import iter_elements
            for i, (idx, _g, L) in enumerate(iter_elements(X, lambda n: n >= 2, msg)):
                if not L:
                    continue  # pack raises the missing-labels error
                try:
                    attributes = np.array(list(L.values()))
                except TypeError:
                    raise TypeError("All attributes of a single graph should have the same dimension.")
                if attributes.ndim != 2 or not np.issubdtype(attributes.dtype, np.number):
                    raise TypeError("GraphHopper needs continuous node attributes: each node label must be a numeric "
                                    "vector, giving an array of shape (n_nodes, n_features) per graph. Got an array of "
                                    "shape " + str(attributes.shape) + " with dtype " + str(attributes.dtype) +
                                    " on the graph at index " + str(i) + ".")
            block = pack(X, "sp", need_labels=True, len_ok=lambda n: n >= 2, want_weights=True,
                         fw_zero_is_absent=True, attributes=True, type_error_msg=msg)
        if block.weights is not None and np.any(np.asarray(block.weights) != 1.0):
            raise NotImplementedError("GraphHopper: edge weights other than 1 are not supported (the shortest-path "
                                      "DAG of the kernel is defined for unweighted graphs)")
        return block

    def parse_input(self, X):
        block = self._pack(X)
        if self._node_kernel is None:
            return self._parse_maps(block)
        return Fitted(block, None, {})

    def _parse_maps(self, block):
        """Callable kernel_type: one (M, attributes) tuple per graph, M from the device (gk_gh_node_maps), zero-padded
        to max(fit delta, this input's delta) like graph_hopper.py:169-172."""
        with _lib.engine(getattr(self, "device_", None)) as eng:
            eng.pack(block.graph_ptr, block.row_ptr, block.col_idx, None, None, block.attrs)
            self.stats_ = eng.gh_features(_lib.GK_GH_LINEAR)
            delta = eng.gh_delta
            if self._method_calling in (1, 2):
                self._max_diam = delta
            width = max(self._max_diam, delta)
            items, gp = [], block.graph_ptr
            for g in range(block.n_graphs):
                n = int(gp[g + 1] - gp[g])
                M = np.zeros((n, width, width))
                if n:
                    M[:, :delta, :delta] = eng.gh_node_maps(g, n)
                items.append((M, np.array(block.attrs[gp[g]:gp[g + 1]], dtype=float)))
        return items

    def pairwise_operation(self, x, y):
        """graph_hopper.py:268-292: both maps truncated to the smaller delta, flattened per vertex."""
        xp, yp = x[0], y[0]
        m = min(xp.shape[1], yp.shape[1])
        xp, yp = xp[:, :m, :m], yp[:, :m, :m]
        return self.metric_((xp.reshape(xp.shape[0], m * m),) + tuple(x[1:]),
                            (yp.reshape(yp.shape[0], m * m),) + tuple(y[1:]))

    # ---- estimator protocol
    def fit(self, X, y=None):
        super().fit(X)
        if self._node_kernel is not None and self._method_calling == 1:
            # delta of the fitted graphs (graph_hopper.py:169-170): one node-map pass on the device
            with _lib.engine(getattr(self, "device_", None)) as eng:
                b = self.X.block
                eng.pack(b.graph_ptr, b.row_ptr, b.col_idx, None, None, b.attrs)
                self._max_diam = int(eng.gh_features(*self._node_kernel).level_dims[0])
        return self

    def fit_transform(self, X, y=None):
        self.initialize()
        if self._node_kernel is None:
            return self._pairwise_fit_transform(X)
        self._method_calling = 2
        self._is_transformed = False
        self.X = self.parse_input(X)
        K, xdiag, _ = self._run(self.X.block, None, n_fit=self.X.block.n_graphs)
        self._max_diam = int(self.stats_.level_dims[0])
        self._X_diag = xdiag
        if self.normalize:
            self._warn_unnormalizable(xdiag)
        return K

    def transform(self, X):
        if self._node_kernel is None:
            return self._pairwise_transform(X)
        self._method_calling = 3
        check_is_fitted(self, ["X"])
        if X is None:
            raise ValueError("`transform` input cannot be None")
        Y = self.parse_input(X)
        K, xdiag, ydiag = self._run(Block.concat(self.X.block, Y.block), None, n_fit=self.X.block.n_graphs)
        self._X_diag = xdiag
        self._Y_diag = ydiag
        self._is_transformed = True
        if self.normalize:
            self._warn_unnormalizable(xdiag, ydiag)
        return K

    def diagonal(self):
        if self._node_kernel is None:
            return self._pairwise_diagonal()
        return super().diagonal()

    def _device_features(self, eng):
        return eng.gh_features(*self._node_kernel)


# ------------------------------------------------------------------------------
_NH_ELEMENT_MSG = ("each element of X must be either a graph object or a list with at least a graph like object and "
                   "node labels dict \n")


class NeighborhoodHash(Kernel):
    """Neighborhood hashing kernel (neighborhood_hash.py:14-570; Hido & Kashima 2009).

    Every label gets a random code of `bits` bits at fit; each of the R levels rehashes every vertex from its own code
    and its out-neighbours' codes ("simple": a rotation XOR-ed with the neighbours' codes, "count_sensitive": one
    rotated term per run of equal codes after a stable sort of the neighbours by their low `bits` bits), and
    K(G, G') = mean over the levels of c / (n + n' - c), c the number of vertex codes the two graphs share (a multiset
    intersection) and n, n' their vertex counts.  The codes, the intersections (an exact integer Gram per level) and
    the fp64 combine run on the device; K equals the reference's bit for bit.

    As in the reference, K is never normalised (`normalize` is accepted and ignored) and `diagonal()` is 1.0.
    Vertices are the symbols of the edge dictionary; the labels of every labelled vertex, also one outside every
    edge, enter the code dictionary.  A label unseen at fit is None in `transform`, and so is every vertex that has it
    or has a neighbour that is None at the previous level.  Deviations: bits > 64 and R > 64 raise
    NotImplementedError; an element with a graph but no labels raises TypeError."""

    _graph_format = "dictionary"

    def __init__(self, n_jobs=None, normalize=False, verbose=False, random_state=None, R=3, nh_type="simple", bits=8):
        super().__init__(n_jobs=n_jobs, normalize=normalize, verbose=verbose)
        self.random_state = random_state
        self.R = R
        self.nh_type = nh_type
        self.bits = bits
        self._initialized.update({"random_state": False, "R": False, "nh_type": False, "bits": False})

    def initialize(self):
        """neighborhood_hash.py:61-89."""
        super().initialize()
        if not self._initialized["random_state"]:
            self.random_state_ = check_random_state(self.random_state)
            self._initialized["random_state"] = True
        if not self._initialized["R"]:
            if type(self.R) is not int or self.R <= 0:
                raise TypeError("R must be an intger bigger than zero")
            if self.R > 64:
                raise NotImplementedError("NeighborhoodHash: at most R = 64 levels are supported")
            self._initialized["R"] = True
        if not self._initialized["nh_type"]:
            if self.nh_type == "simple":
                self._nh_code = _lib.GK_NH_SIMPLE
            elif self.nh_type == "count_sensitive":
                self._nh_code = _lib.GK_NH_COUNT_SENSITIVE
            else:
                raise TypeError("unrecognised neighborhood hashing type")
            self._initialized["nh_type"] = True
        if not self._initialized["bits"]:
            if type(self.bits) is not int or self.bits <= 0:
                raise TypeError("illegal number of bits for hashing")
            if self.bits > 64:
                raise NotImplementedError("NeighborhoodHash: codes are 64-bit on the device; bits > 64 is not supported")
            self._max_number = 1 << self.bits
            self._mask = self._max_number - 1
            self._initialized["bits"] = True

    # ---- input
    @staticmethod
    def _elements(X):
        """[graph, node labels] of every element, with the reference's element checks (neighborhood_hash.py:123-151)."""
        if not isinstance(X, Iterable):
            raise TypeError("input must be an iterable\n")
        out = []
        for idx, x in enumerate(iter(X)):
            if isinstance(x, Graph):
                x = x.as_element()
            is_iter = isinstance(x, Iterable)
            if is_iter:
                x = list(x)
            if not (is_iter and len(x) in (0, 1, 2, 3)):
                raise TypeError(_NH_ELEMENT_MSG)
            if len(x) == 0:
                warnings.warn("Ignoring empty element on index: " + str(idx))
                continue
            if len(x) == 1:
                raise TypeError("Ignoring empty element on index: " + str(len(out)) + "\nLabels must be provided.")
            if type(x[0]) is dict and x[0] and all(type(d) is list for d in x[0].values()) and not all(x[0].values()):
                # {u: []}: u is a vertex without an edge-dictionary entry (graph.py:1634-1650, 849-855)
                raise ValueError("vertex not inside edge dictionary")
            out.append([x[0], x[1]])
        return out

    @staticmethod
    def _from_packed(X):
        """A read_tu(kernel="NH") block holds every labelled node (all of their labels enter the code dictionary);
        the kernel's vertex set is the nodes that occur in an edge (graph.py:1613-1703).  The neighbour order of the
        reference's edge sets (read_data builds Python sets, base.py:215-222) is not known here; `_nh_run` refuses a
        count-sensitive result that depends on it."""
        X.require("wl")
        labels = np.asarray(X.labels)
        gp0 = np.asarray(X.graph_ptr, dtype=np.int64)
        values = [labels[gp0[g]:gp0[g + 1]].tolist() for g in range(X.n_graphs)]
        rp = np.asarray(X.row_ptr, dtype=np.int64)
        ci = np.asarray(X.col_idx, dtype=np.int64)
        deg = np.diff(rp)
        keep = deg > 0
        keep[ci] = True
        before = np.concatenate([[0], np.cumsum(keep)])
        block = Block(before[gp0], np.concatenate([[0], np.cumsum(deg[keep])]), before[ci], None, labels[keep])
        block.mode = "sp"
        return block, values

    def parse_input(self, X):
        fit = self._method_calling in (1, 2)
        if isinstance(X, Block) and X.mode == "core":  # a CoreFramework level: every vertex, neighbours in order
            block, gp = X, X.graph_ptr
            values = [X.labels[gp[g]:gp[g + 1]] for g in range(X.n_graphs)]
        elif isinstance(X, Block):
            block, values = self._from_packed(X)
        else:
            els = self._elements(X)
            block = pack(els, "sp", need_labels=True, len_ok=lambda n: n == 2, type_error_msg=_NH_ELEMENT_MSG,
                         keep_edge_order=True)
            values = [list(L.values()) for _, L in els]
        if fit:  # neighborhood_hash.py:157-189: the label set and the draws, operation for operation
            labels_hash_set = set()
            for vals in values:
                labels_hash_set |= set(vals)
            if len(labels_hash_set) > self._max_number:
                warnings.warn("Number of labels is smaller than"
                              "the biggest possible.. "
                              "Collisions will appear on the "
                              "new labels.")
                nl, nrl = list(), len(labels_hash_set)
                while nrl > self._max_number:
                    nl += self.random_state_.choice(self._max_number, self._max_number, replace=False).tolist()
                    nrl -= self._max_number
                if nrl > 0:
                    nl += self.random_state_.choice(self._max_number, nrl, replace=False).tolist()
            else:
                nl = self.random_state_.choice(self._max_number, len(labels_hash_set), replace=False).tolist()
            self._labels_hash_dict = dict(zip(labels_hash_set, nl))
        ids, dictionary = label_ids(block.labels, None, sort_new=False)
        hd = self._labels_hash_dict
        fitted = Fitted(block, ids, dictionary)
        fitted.order_known = not isinstance(X, Block) or X.mode == "core"
        fitted.codes = np.array([hd.get(l, 0) for l in dictionary], dtype=np.uint64)
        fitted.valid = np.array([l in hd for l in dictionary], dtype=np.uint8)
        return fitted

    # ---- estimator protocol
    def fit(self, X, y=None):
        self._method_calling = 1
        self._is_transformed = False
        self.initialize()
        if X is None:
            raise ValueError("`fit` input cannot be None")
        self.X = self.parse_input(X)
        return self

    def fit_transform(self, X, y=None):
        self._method_calling = 2
        self.fit(X)
        b = self.X.block
        if np.any(np.diff(b.graph_ptr) == 0):  # nh_compare_labels of two vertex-less graphs: 0 / 0
            raise ZeroDivisionError("float division by zero")
        return self._nh_run(b, self.X.ids, self.X.codes, self.X.valid, b.n_graphs, self.X.order_known)

    def transform(self, X):
        self._method_calling = 3
        check_is_fitted(self, ["X"])
        if X is None:
            raise ValueError("`transform` input cannot be None")
        Y = self.parse_input(X)
        xb = self.X.block
        if np.any(np.diff(xb.graph_ptr) == 0) and np.any(np.diff(Y.block.graph_ptr) == 0):
            raise ZeroDivisionError("float division by zero")
        K = self._nh_run(Block.concat(xb, Y.block), np.concatenate([self.X.ids, Y.ids + len(self.X.codes)]),
                         np.concatenate([self.X.codes, Y.codes]), np.concatenate([self.X.valid, Y.valid]), xb.n_graphs,
                         self.X.order_known and Y.order_known)
        self._is_transformed = True
        return K

    def diagonal(self):
        """neighborhood_hash.py:343-365: the kernel's self similarities are 1."""
        if self._is_transformed:
            return 1.0, 1.0
        return 1.0

    def _nh_run(self, block, ids, codes, valid, n_fit, order_known=True):
        """pack -> gk_nh_features (R hash levels, per-level columns) -> gk_gram (per-level Grams, fp64 combine).
        `order_known`: the block's rows list every vertex's neighbours in the reference's edge-dictionary order."""
        with _run_engine(self) as eng:
            eng.pack(block.graph_ptr, block.row_ptr, block.col_idx, ids, None, None)
            self.stats_ = eng.nh_features(self.R, self._nh_code, self.bits, codes, valid)
            if self.stats_.nh_order_dependent and not order_known:
                raise NotImplementedError(
                    "NeighborhoodHash(nh_type='count_sensitive'): a vertex has two different neighbour codes with equal "
                    "low bits, so its code depends on the neighbour order of the reference's edge sets, which a packed "
                    "block does not carry; pass the list of graphs instead")
            K, _, _ = _gram_or_fold(self, eng, block.n_graphs, n_fit, stats=self.stats_, want_diag=False)
        if self.verbose:
            print(type(self).__name__, self.stats_.as_dict())
        return K


# ------------------------------------------------------------------------------
def _stacked_by_size(mats, fn):
    """fn over every matrix of `mats`, called once per vertex count on the stacked (k, n, n) array: numpy's LAPACK
    gufuncs run the same routine matrix by matrix, so the results equal per-matrix calls bit for bit."""
    out = [None] * len(mats)
    groups = {}
    for i, A in enumerate(mats):
        groups.setdefault(A.shape[0], []).append(i)
    for n, idx in groups.items():
        if n == 0:
            for i in idx:
                out[i] = None
            continue
        res = fn(np.stack([mats[i] for i in idx]))
        for k, i in enumerate(idx):
            out[i] = tuple(r[k] for r in res) if isinstance(res, tuple) else res[k]
    return out


def spectral_radii(mats):
    """random_walk.py:139-144 (largest |eigenvalue| of numpy.linalg.eigvals, 0 for an empty graph), stacked by size."""
    ev = _stacked_by_size(mats, np.linalg.eigvals)
    return [0.0 if e is None else float(np.max(np.absolute(e))) for e in ev]


def _eigen_data(mats, symmetric):
    """Per-vertex (q, w) of every graph, concatenated: (real(1^T V), real(w)) of numpy.linalg.eig as the reference's
    `sd` (random_walk.py:548-553), or of numpy.linalg.eigh for the symmetric inverse."""
    res = _stacked_by_size(mats, np.linalg.eigh if symmetric else np.linalg.eig)
    qs, ws = [], []
    for r in res:
        if r is None:
            continue
        w, v = r
        qs.append(np.real(np.sum(v, axis=0)))
        ws.append(np.real(w))
    if not qs:
        return np.zeros(0), np.zeros(0)
    return np.concatenate(qs), np.concatenate(ws)


def _block_adjacency(X, labeled):
    """(adjacency matrix, labels or None) of every graph of a datasets.read_tu block: the kernel's vertices are the
    nodes that occur in an edge (the reference's adjacency matrix of an edge-set graph)."""
    X.require("sp", labels=labeled)
    out = []
    gp, rp, ci = X.graph_ptr, X.row_ptr, X.col_idx
    for g in range(X.n_graphs):
        a, b = int(gp[g]), int(gp[g + 1])
        A = np.zeros((b - a, b - a))
        for u in range(a, b):
            e0, e1 = int(rp[u]), int(rp[u + 1])
            A[u - a, ci[e0:e1] - a] = 1.0 if X.weights is None else X.weights[e0:e1]
        out.append((A, list(X.labels[a:b]) if labeled else None))
    return out


_RW_ELEMENT_MSG = "each element of X must be either a graph or an iterable with at least 1 and at most 3 elements\n"
_RWL_ELEMENT_MSG = "each element of X must be either a graph or an iterable with at least 2 and at most 3 elements\n"


class RandomWalk(Kernel):
    """Random walk kernel (random_walk.py:28-341; Gaertner et al. 2003, Vishwanathan et al. 2010).

    Same parameters, attributes (`mu_`, `_lamda`), errors and warnings as the reference, including the lowering of
    lamda at fit time when the geometric series would diverge.  Every pair runs on the device in fp64:
    method_type="fast" with the geometric kernel replays scipy's conjugate gradients per pair; the fast spectral
    variants and the baseline geometric kernel on symmetric matrices sum over the eigen-pairs of both graphs (computed on
    the host with numpy, as the reference does); the baseline finite series and exponential run as power series of
    matvecs.  The baseline geometric kernel of a non-symmetric matrix raises NotImplementedError, as does the baseline
    exponential kernel on a matrix with a negative entry."""

    _graph_format = "adjacency"
    _labeled = False

    def __init__(self, n_jobs=None, normalize=False, verbose=False, lamda=0.1, method_type="fast",
                 kernel_type="geometric", p=None):
        super().__init__(n_jobs=n_jobs, normalize=normalize, verbose=verbose)
        self.method_type = method_type
        self.kernel_type = kernel_type
        self.p = p
        self.lamda = lamda
        self._initialized.update({"method_type": False, "kernel_type": False, "p": False, "lamda": False})

    def initialize(self):
        """random_walk.py:81-133, in its order: method_type, kernel_type, p (mu_), lamda."""
        super().initialize()
        if not self._initialized["method_type"]:
            if self.method_type not in ("baseline", "fast"):
                raise ValueError("unsupported method_type")
            self._initialized["method_type"] = True
        if not self._initialized["kernel_type"]:
            if self.kernel_type not in ["geometric", "exponential"]:
                raise ValueError('unsupported kernel type: either "geometric" or "exponential"')
        if not self._initialized["p"]:
            if self.p is not None:
                if type(self.p) is int and self.p > 0:
                    self.mu_ = [1]
                    fact, power = 1, 1
                    for k in range(1, self.p + 1):
                        power *= self.lamda
                        if self.kernel_type == "exponential":
                            fact *= k
                            self.mu_.append(power / fact)
                        else:
                            self.mu_.append(power)
                else:
                    raise TypeError("p must be a positive integer bigger than zero or nonetype")
                self._initialized["kernel_type"] = True
        if not self._initialized["lamda"]:
            if self.lamda <= 0:
                raise TypeError("lambda must be positive bigger than equal")
            self._lamda = self.lamda
            self._initialized["lamda"] = True

    _lamda_safety = 0.9

    def _tune_lamda(self, spectral_radii):
        """random_walk.py:146-194: keep the geometric series convergent on the graphs given."""
        if self.kernel_type != "geometric" or self.p is not None:
            return
        if not spectral_radii:
            return
        rho = max(spectral_radii)
        if rho <= 0:
            return
        limit = 1.0 / (rho ** 2)
        if self._method_calling in (1, 2):
            if self.lamda >= limit:
                self._lamda = self._lamda_safety * limit
                warnings.warn(
                    'lamda=' + repr(self.lamda) + ' makes the random walk '
                    'series diverge on these graphs, whose largest spectral '
                    'radius is ' + format(rho, '.4g') + ': convergence needs '
                    'lamda < ' + format(limit, '.4g') + '. Using lamda=' +
                    format(self._lamda, '.4g') + ' instead. Pass a smaller '
                    'lamda, or p=<int> for a fixed number of steps, to '
                    'silence this.', RuntimeWarning)
        else:
            if self._lamda >= limit:
                warnings.warn(
                    'the graphs passed to transform have a larger spectral '
                    'radius (' + format(rho, '.4g') + ') than the fitted '
                    'ones, so lamda=' + format(self._lamda, '.4g') + ' no '
                    'longer converges on them (it needs to stay below ' +
                    format(limit, '.4g') + '). Refit with a smaller lamda: it '
                    'cannot be changed now without invalidating the fit.',
                    RuntimeWarning)

    def _warn_unnormalizable(self, *diagonals):
        """kernel.py:206-234, with the negative-self-similarity message written for the random walk kernels."""
        name = type(self).__name__
        for d in diagonals:
            d = np.asarray(d, dtype=float)
            if np.any(d < 0):
                warnings.warn(
                    name + ' has negative self similarities, so normalizing '
                    'it yields NaNs: k(G, G) < 0 means the kernel is not '
                    'positive semi-definite on this input. For the random '
                    'walk kernels this usually means the decay factor is too '
                    'large for these graphs -- it has to stay below 1 over '
                    'the largest eigenvalue of the product graph adjacency '
                    'matrix. Either lower it or pass normalize=False.',
                    RuntimeWarning)
                break
            if np.any(d == 0):
                warnings.warn(
                    name + ' has zero self similarities, so normalizing it '
                    'yields NaNs: those graphs have no features this kernel '
                    'can see. Either drop them or pass normalize=False.',
                    RuntimeWarning)
                break

    # ---- route
    def _route(self):
        """(route, fn) of random_walk.py:272-341 (RandomWalkLabeled: :491-541)."""
        fast, geo = self.method_type == "fast", self.kernel_type == "geometric"
        if self._labeled:
            if fast and geo and self.p is None:
                return _lib.GK_RW_CG, _lib.GK_RW_INV
            if self.p is not None:
                return _lib.GK_RW_SERIES, _lib.GK_RW_FINITE
            if not geo:
                return _lib.GK_RW_SERIES, _lib.GK_RW_EXP
            raise NotImplementedError("RandomWalkLabeled(method_type='baseline', kernel_type='geometric', p=None): the "
                                      "inverse of the product graph matrix is not computed on the device")
        if fast:
            if self.p is None and geo:
                return _lib.GK_RW_CG, _lib.GK_RW_INV
            return _lib.GK_RW_SPECTRAL, (_lib.GK_RW_FINITE if self.p is not None else _lib.GK_RW_EXP)
        if self.p is not None:
            return _lib.GK_RW_SERIES, _lib.GK_RW_FINITE
        if not geo:
            return _lib.GK_RW_SERIES, _lib.GK_RW_EXP
        return _lib.GK_RW_SPECTRAL, _lib.GK_RW_INV

    # ---- input
    def _elements(self, X):
        """(adjacency matrix, labels in index order or None) of every element (random_walk.py:215-244, 423-448)."""
        from .packing import adjacency_and_labels
        if isinstance(X, Block):
            return _block_adjacency(X, self._labeled)
        if not isinstance(X, Iterable):
            raise TypeError("input must be an iterable\n")
        out = []
        for idx, x in enumerate(iter(X)):
            if isinstance(x, Graph):
                x = x.as_element()
            is_iter = isinstance(x, Iterable)
            if is_iter:
                x = list(x)
            ok = (1, 2, 3) if self._labeled else (0, 1, 2, 3)
            if not (is_iter and len(x) in ok):
                raise TypeError(_RWL_ELEMENT_MSG if self._labeled else _RW_ELEMENT_MSG)
            if len(x) == 0:
                warnings.warn("Ignoring empty element on index: " + str(idx))
                continue
            out.append(adjacency_and_labels(x[0], x[1] if self._labeled else None))
        if not out:
            raise ValueError("parsed input is empty")
        return out

    def parse_input(self, X):
        import time
        els = self._elements(X)
        mats = [A for A, _ in els]
        t0 = time.perf_counter()
        if self.kernel_type == "geometric" and self.p is None:
            self._tune_lamda(spectral_radii(mats))
        route, fn = self._route()
        fitted = Fitted(None, None, {})
        fitted.mats = mats
        fitted.labels = [L for _, L in els]
        fitted.q = fitted.w = None
        if route == _lib.GK_RW_SPECTRAL:
            symmetric = fn == _lib.GK_RW_INV
            if symmetric and not all(np.array_equal(A, A.T) for A in mats):
                raise NotImplementedError("RandomWalk(method_type='baseline', kernel_type='geometric', p=None) is "
                                          "computed from the eigen-decomposition of symmetric adjacency matrices only")
            fitted.q, fitted.w = _eigen_data(mats, symmetric)
        elif route == _lib.GK_RW_SERIES and fn == _lib.GK_RW_EXP and any(np.any(A < 0) for A in mats):
            raise NotImplementedError("the baseline exponential random walk kernel is summed as a power series, which "
                                      "needs non-negative adjacency entries")
        self.ms_host_eig_ = (time.perf_counter() - t0) * 1e3
        return fitted

    @staticmethod
    def _concat(a, b):
        out = Fitted(None, None, {})
        out.mats = a.mats + b.mats
        out.labels = a.labels + b.labels
        out.q = None if a.q is None else np.concatenate([a.q, b.q])
        out.w = None if a.w is None else np.concatenate([a.w, b.w])
        return out

    # ---- estimator protocol
    def fit_transform(self, X, y=None):
        self._method_calling = 2
        self.fit(X)
        K, xdiag, _ = self._rw_run(self.X, len(self.X.mats))
        self._X_diag = xdiag
        if self.normalize:
            self._warn_unnormalizable(xdiag)
        return K

    def transform(self, X):
        self._method_calling = 3
        check_is_fitted(self, ["X"])
        if X is None:
            raise ValueError("`transform` input cannot be None")
        Y = self.parse_input(X)
        K, xdiag, ydiag = self._rw_run(self._concat(self.X, Y), len(self.X.mats))
        self._X_diag, self._Y_diag = xdiag, ydiag
        self._is_transformed = True
        if self.normalize:
            self._warn_unnormalizable(xdiag, ydiag)
        return K

    def diagonal(self):
        check_is_fitted(self, ["X"])
        try:
            check_is_fitted(self, ["_X_diag"])
        except NotFittedError:
            _, self._X_diag, _ = self._rw_run(self.X, len(self.X.mats), want_matrix=False)
        if getattr(self, "_is_transformed", False):
            return self._X_diag, self._Y_diag
        return self._X_diag

    def _rw_run(self, data, n_fit, want_matrix=True, device_ptr=None):
        """pack the structure -> gk_rw_features -> gk_gram.  Returns (K, xdiag, ydiag)."""
        route, fn = self._route()
        mats = data.mats
        sizes = np.array([A.shape[0] for A in mats], dtype=np.int64)
        gp = np.concatenate([[0], np.cumsum(sizes)])
        rows, cols, vals, trows, tcols, tvals = [], [], [], [], [], []
        for g, A in enumerate(mats):
            ii, jj = np.nonzero(A)
            rows.append(ii + gp[g]); cols.append(jj + gp[g]); vals.append(A[ii, jj])
            ti, tj = np.nonzero(A.T)
            trows.append(ti + gp[g]); tcols.append(tj + gp[g]); tvals.append(A.T[ti, tj])
        cat = lambda parts, dt: np.concatenate(parts).astype(dt) if parts else np.zeros(0, dt)
        V = int(gp[-1])
        r, c, v = cat(rows, np.int64), cat(cols, np.int32), cat(vals, np.float64)
        tr, tc, tv = cat(trows, np.int64), cat(tcols, np.int32), cat(tvals, np.float64)
        rp = np.concatenate([[0], np.cumsum(np.bincount(r, minlength=V))])
        trp = np.concatenate([[0], np.cumsum(np.bincount(tr, minlength=V))])
        ids = None
        if self._labeled:
            ids, _ = label_ids([l for L in data.labels for l in L], None, sort_new=False)
        coef = self.mu_ if fn == _lib.GK_RW_FINITE else None
        with _lib.engine(getattr(self, "device_", None)) as eng:
            eng.pack(gp, rp, c, ids, None, None)
            eng.rw_features(route, fn, self._lamda, coef, v, trp, tc, tv, data.q, data.w, labeled=self._labeled)
            self.stats_ = _lib.GkStats()
            out = False if not want_matrix else None
            K, xd, yd = eng.gram(len(mats), n_fit=n_fit, normalize=bool(self.normalize) and want_matrix,
                                 out=out if device_ptr is None else None, device_ptr=device_ptr, stats=self.stats_)
        if self.verbose:
            print(type(self).__name__, self.stats_.as_dict())
        return K, xd, yd


class RandomWalkLabeled(RandomWalk):
    """Labelled random walk kernel (random_walk.py:343-541): walks of the product graph pair vertices with equal labels.
    Conjugate gradients for the fast geometric kernel, power series for the finite and exponential variants; the
    baseline geometric kernel with p=None raises NotImplementedError."""

    _labeled = True


# ------------------------------------------------------------------------------
def _pk_dot(x, y):
    """propagation.py:23-24: the default metric, a dot product of two Counters."""
    return sum(x[k] * y[k] for k in x)


def row_normalized(mats):
    """sklearn's normalize(T, axis=1, norm="l1") of every matrix (propagation.py:220, 568).  Dense matrices of one shape
    and dtype go through one call on their vertical stack: the l1 norms and the division are row by row, so every block
    of the result equals the per-matrix call bit for bit.  Only C-ordered matrices are stacked (numpy sums a strided
    row in another order than a contiguous one); anything else is normalised matrix by matrix."""
    from sklearn.preprocessing import normalize
    out = [None] * len(mats)
    groups = {}
    for i, T in enumerate(mats):
        if isinstance(T, np.ndarray) and T.ndim == 2 and T.shape[0] > 0 and T.flags.c_contiguous:
            groups.setdefault((T.shape, T.dtype.str), []).append(i)
        else:
            out[i] = normalize(T, axis=1, norm="l1")
    for (shape, _), idx in groups.items():
        stacked = normalize(np.vstack([mats[i] for i in idx]), axis=1, norm="l1")
        for k, i in enumerate(idx):
            out[i] = stacked[k * shape[0]:(k + 1) * shape[0]]
    return out


_PK_ELEMENT_MSG = "Each element of X must be either a Graph or an iterable with at least 2 and at most 4 elements\n"


class Propagation(Kernel):
    """Propagation kernel for labelled graphs (propagation.py:27-423; Neumann et al. 2016).

    Every vertex starts as the one-hot vector of its label; at each of t_max levels it is hashed into a bin,
    floor((P_v . u_t + b_t) / w) with random u_t (Gaussian, or Cauchy for M="TV") and b_t drawn at fit, and every graph
    then propagates P <- T P with its row-normalised transition matrix T (the adjacency matrix, or a matrix given as
    the element's 4th entry).  K(G, G') = sum_t sum_c n_t(G, c) n_t(G', c), n_t(G, c) the vertices of G in bin c at
    level t.  Propagation, hashing and the exact integer Gram run on the device; the label set, the draws and the
    normalisation of T are the reference's own operations in its order.

    Parameters, fitted attributes (`random_state_`, `_u`, `_b`, `_enum_labels`, `_parent_labels`) and errors are the
    reference's, quirks included (a non-callable `metric` is not rejected; w < 0 is accepted).  A transform whose
    graphs carry labels unseen at fit follows the reference's second branch: fresh draws per level for the new labels,
    private bins for the vertices that hash with them, and the reference's inclusive count of each graph's successor's
    first vertex.  `stats_.pk_near_edge` counts the hashes that lie within 2^-30 of their magnitude of a bin edge:
    only those can fall into another bin than the reference's, whose summation order may differ.

    A callable `metric` gets the reference's per-level Counters, built from the device bins with the reference's id
    assignment, through the generic pairwise driver; `_hd` is built the same way on first access.

    Deviations: w == 0 and t_max > 64 raise NotImplementedError; a NaN bin (M="H" over a negative entry) raises
    KeyError as the reference does, but from the device check.  A sparse transition matrix raises the reference's
    ValueError when t_max > 1."""

    _graph_format = "adjacency"
    attr_ = False

    def __init__(self, n_jobs=None, verbose=False, normalize=False, random_state=None, metric=_pk_dot, M="TV", t_max=5,
                 w=0.01):
        super().__init__(n_jobs=n_jobs, verbose=verbose, normalize=normalize)
        self.random_state = random_state
        self.M = M
        self.t_max = t_max
        self.w = w
        self.metric = metric
        self._initialized.update({"M": False, "t_max": False, "w": False, "random_state": False, "metric": False})

    def initialize(self):
        """propagation.py:93-131, in its order and with its quirks."""
        super().initialize()
        if not self._initialized["random_state"]:
            self.random_state_ = check_random_state(self.random_state)
            self._initialized["random_state"] = True
        if not self._initialized["metric"]:
            if (type(self.M) is not str or (self.M not in ["H", "TV"] and not self.attr_)
                    or (self.M not in ["L1", "L2"] and self.attr_)):
                if self.attr_:
                    raise TypeError('Metric type must be a str, one of "L1", "L2"')
                raise TypeError('Metric type must be a str, one of "H", "TV"')
            if not self.attr_:
                self.take_sqrt_ = self.M == "H"
            self.take_cauchy_ = self.M in ["TV", "L1"]
            self._initialized["metric"] = True
        if not self._initialized["t_max"]:
            if type(self.t_max) is not int or self.t_max <= 0:
                raise TypeError("The number of iterations must be a positive integer.")
            if self.t_max > 64:
                raise NotImplementedError(type(self).__name__ + ": at most t_max = 64 levels are supported")
            self._initialized["t_max"] = True
        if not self._initialized["w"]:
            if not isinstance(self.w, Real) and self.w <= 0:
                raise TypeError("The bin width must be a positive number.")
            if self.w == 0:
                raise NotImplementedError(type(self).__name__ + ": w = 0 puts every vertex into an infinite bin; "
                                          "pass a non-zero bin width")
            self._initialized["w"] = True
        if not self._initialized["metric"]:
            if not callable(self.metric):
                raise TypeError("The base kernel must be callable.")
            self._initialized["metric"] = True

    # ---- input
    def _elements(self, X, check=None):
        """(adjacency matrix, labels / attributes in index order, T or None) of every element (propagation.py:169-226).
        `check(lab)` validates an element's labels.  The reference normalises each element's T before checking its
        labels, element by element; T is normalised in groups here, so an error raised for element k first lets the
        normalisation of the elements before it (and of element k, for a label error) raise its own error."""
        from .packing import adjacency_and_labels
        if isinstance(X, Block):  # datasets.read_tu: the kernel's vertices are the nodes that occur in an edge
            X.require("sp", labels=not self.attr_)
            out = []
            gp, rp, ci = X.graph_ptr, X.row_ptr, X.col_idx
            for g in range(X.n_graphs):
                a, b = int(gp[g]), int(gp[g + 1])
                A = np.zeros((b - a, b - a))
                for v in range(a, b):
                    e0, e1 = int(rp[v]), int(rp[v + 1])
                    A[v - a, ci[e0:e1] - a] = 1.0 if X.weights is None else X.weights[e0:e1]
                lab = list(np.asarray(X.attrs)[a:b]) if self.attr_ else list(X.labels[a:b])
                if check:
                    check(lab)
                out.append((A, lab, None))
            return out
        if not isinstance(X, Iterable):
            raise ValueError("input must be an iterable\n")
        out = []

        def normalised_first(err, upto):
            row_normalized([A if T is None else T for A, _, T in out[:upto]])
            raise err

        for idx, x in enumerate(iter(X)):
            is_iter = isinstance(x, Iterable)
            if is_iter and not isinstance(x, Graph):
                x = list(x)
            if is_iter and not isinstance(x, Graph) and len(x) in [0, 2, 3, 4]:
                if len(x) == 0:
                    warnings.warn("Ignoring empty element on " + "index: " + str(idx))
                    continue
                if len(x) == 2 and isinstance(x[0], Graph):
                    el, T = x[0].as_element(), x[1]
                else:
                    el, T = x, (x[3] if len(x) == 4 else None)
            elif isinstance(x, Graph):
                el, T = x.as_element(), None
            else:
                normalised_first(ValueError("Each element of X must be either a " + "Graph or an iterable with at "
                                            "least 2 " + "and at most 4 elements\n"), len(out))
            try:
                A, lab = adjacency_and_labels(el[0], el[1])
                if T is not None:
                    if T.shape[0] != T.shape[1]:
                        raise TypeError("Transition matrix on index" + " " + str(idx) + "must be " +
                                        "a square matrix.")
                    if T.shape[0] != A.shape[0]:
                        raise TypeError("Propagation matrix must " + "have the same dimension " +
                                        "as the number of vertices.")
            except Exception as e:  # noqa: BLE001
                normalised_first(e, len(out))
            out.append((A, lab, T))
            if check:
                try:
                    check(lab)
                except Exception as e:  # noqa: BLE001
                    normalised_first(e, len(out))
        return out

    def _transitions(self, els):
        """Row-normalised T of every element as dense float64 (the values numpy's dot reads), and whether one of them
        is a scipy sparse matrix (numpy's dot cannot propagate it: propagation.py:292 raises at the first step)."""
        normed = row_normalized([A if T is None else T for A, _, T in els])
        out, sparse = [], False
        for T in normed:
            if not isinstance(T, np.ndarray):
                sparse = True
                T = T.toarray()
            out.append(np.asarray(T, dtype=np.float64))
        return out, sparse

    def _sparse_step_error(self, data):
        """The reference's error at its first propagation step over a sparse T, raised where it raises it: after the
        draws of the fit, or after the first level's draws of a transform with new labels."""
        if data.sparse and self.t_max > 1:
            raise ValueError("setting an array element with a sequence.")

    def parse_input(self, X):
        """propagation.py:149-294: the label set, the enumeration and the draws, operation for operation."""
        labels = set()

        def check(lab):
            nonlocal labels
            try:
                labels |= set(lab)
            except TypeError:
                raise TypeError("For a non attributed kernel, labels should be hashable.")

        els = self._elements(X, check)
        if not els:
            raise ValueError("Parsed input is empty")
        data = Fitted(None, None, {})
        data.T, data.sparse = self._transitions(els)
        data.sizes = np.array([len(lab) for _, lab, _ in els], dtype=np.int64)
        data.u_full = None
        if self._method_calling == 1:
            enum_labels = {l: i for (i, l) in enumerate(list(labels))}
            self._enum_labels = enum_labels
            self._parent_labels = labels
        else:
            new_elements = labels - self._parent_labels
            if len(new_elements) > 0:
                new_enum_labels = iter((l, i) for (i, l) in enumerate(list(new_elements), len(self._enum_labels)))
                enum_labels = dict(chain(self._enum_labels.items(), new_enum_labels))
            else:
                enum_labels = self._enum_labels
        data.ids = np.array([enum_labels[l] for _, lab, _ in els for l in lab], dtype=np.int32)
        data.dim = len(enum_labels)
        dim_orig = len(self._enum_labels)
        if self._method_calling == 1:
            self._u, self._b = list(), list()
            for t in range(self.t_max):
                u = self.random_state_.randn(len(enum_labels))
                if self.take_cauchy_:
                    u = np.divide(u, self.random_state_.randn(len(enum_labels)))
                self._u.append(u)
                self._b.append(self.w * self.random_state_.rand())
            self._hd_cache = None
        elif dim_orig < len(enum_labels):  # :353-359, drawn level by level at transform time
            nnv = len(enum_labels) - dim_orig
            data.u_full = []
            for t in range(self.t_max if not (data.sparse and self.t_max > 1) else 1):
                u = self.random_state_.randn(nnv)
                if self.take_cauchy_:
                    u = np.divide(u, self.random_state_.randn(nnv))
                data.u_full.append(np.hstack((self._u[t], u)))
        self._sparse_step_error(data)
        return data

    # ---- estimator protocol
    def _default_metric(self):
        return self.metric is _pk_dot

    def pairwise_operation(self, x, y):
        """propagation.py:133-147: the metric summed over the levels' Counters."""
        return sum(self.metric(x[t], y[t]) for t in range(self.t_max))

    def fit_transform(self, X, y=None):
        self._method_calling = 2
        self.fit(X)
        if not self._default_metric():
            return self._metric_fit_transform()
        K, xdiag, _ = self._pk_run(self.X, None, want_matrix=True)
        self._X_diag = xdiag
        if self.normalize:
            self._warn_unnormalizable(xdiag)
        return K

    def transform(self, X):
        self._method_calling = 3
        check_is_fitted(self, ["X"])
        if X is None:
            raise ValueError("`transform` input cannot be None")
        Y = self.parse_input(X)
        if not self._default_metric():
            return self._metric_transform(Y)
        K, xdiag, ydiag = self._pk_run(self.X, Y, want_matrix=True)
        self._X_diag, self._Y_diag = xdiag, ydiag
        self._is_transformed = True
        if self.normalize:
            self._warn_unnormalizable(xdiag, ydiag)
        return K

    def diagonal(self):
        check_is_fitted(self, ["X"])
        if not self._default_metric():
            return self._with_phi(self._pairwise_diagonal)
        try:
            check_is_fitted(self, ["_X_diag"])
        except NotFittedError:
            _, self._X_diag, _ = self._pk_run(self.X, None, want_matrix=False)
        if getattr(self, "_is_transformed", False):
            return self._X_diag, self._Y_diag
        return self._X_diag

    # ---- callable metric: the reference's Counters from the device bins, through the generic pairwise driver
    @property
    def _hd(self):
        """The fit's per-level bin -> id dictionaries (propagation.py:280, 615), built lazily from the device bins of
        the fitted graphs with the reference's id assignment."""
        check_is_fitted(self, ["X"])
        if getattr(self, "_hd_cache", None) is None:
            levels = self._device_bins(self.X, None)
            self._hd_cache = [self._fit_ids(b)[0] for b, _ in levels]
        return self._hd_cache

    def _device_bins(self, X, Y):
        """Per level (bins [V, K], private flags [V]) of the joint X || Y block."""
        with _lib.engine(getattr(self, "device_", None)) as eng:
            self.stats_, V, _, _ = self._pk_features(eng, X, Y)
            width = self._dim if self.attr_ else 1
            return [eng.pk_hashes(t, V, width) for t in range(self.t_max)]

    def _fit_ids(self, bins):
        """(hd, ids) of one level at fit (propagation.py:279-282; attributes :613-618)."""
        if self.attr_:
            hashes = bins.tolist()
            hd = {j: i for i, j in enumerate({tuple(l) for l in hashes})}
            return hd, np.array([hd[tuple(l)] for l in hashes])
        hashes = bins[:, 0]
        hd = dict((j, i) for i, j in enumerate(set(np.unique(hashes))))
        return hd, np.vectorize(lambda i: hd[i])(hashes)

    def _transform_ids(self, hd_fit, bins, otypes=None):
        """ids of one level's transformed bins: the fit's ids, then fresh ids in the reference's order
        (propagation.py:301-314, 338-351; attributes :638-653)."""
        if self.attr_:
            hashes = bins.tolist()
            new = filterfalse(lambda x: x in hd_fit, {tuple(l) for l in hashes})
            hd = dict(chain(hd_fit.items(), ((j, i) for i, j in enumerate(new, len(hd_fit)))))
            return hd, np.array([hd[tuple(l)] for l in hashes])
        hashes = bins[:, 0]
        new = filterfalse(lambda x: x in hd_fit, np.unique(hashes))
        hd = dict(chain(hd_fit.items(), ((j, i) for i, j in enumerate(new, len(hd_fit)))))
        if len(hashes) == 0:
            return hd, np.zeros(0, dtype=int)
        return hd, np.vectorize(lambda i: hd[i], otypes=otypes)(hashes)

    def _phi(self, levels, sizes, offset, hd_fit=None, split=False):
        """The reference's per-graph {level: Counter} of the graphs whose vertices start at `offset`: ids assigned as at
        fit (hd_fit None) or as at transform, `split` for a transform with labels unseen at fit (ordinary and private
        vertices, propagation.py:328-395)."""
        idx = np.concatenate([[0], np.cumsum(sizes)])
        n, V = len(sizes), int(idx[-1])
        phi = [dict() for _ in range(n)]
        for t, (bins, priv) in enumerate(levels):
            b, pv = bins[offset:offset + V], priv[offset:offset + V]
            if hd_fit is None:
                _, features = self._fit_ids(b)
            elif not split:
                _, features = self._transform_ids(hd_fit[t], b)
            else:
                vertices, vertices_p = np.where(~pv)[0], np.where(pv)[0]
                hd, features = self._transform_ids(hd_fit[t], b[vertices], otypes=[int])
                hashes = b[vertices_p, 0]
                hd = dict(chain(hd.items(), ((j, i) for i, j in enumerate(hashes, len(hd)))))
                features_p = np.vectorize(lambda i: hd[i], otypes=[int])(hashes) if len(hashes) else \
                    np.zeros(0, dtype=int)
                for k in range(n):
                    A = Counter(features[np.logical_and(idx[k] <= vertices, vertices <= idx[k + 1])])
                    B = Counter(features_p[np.logical_and(idx[k] <= vertices_p, vertices_p <= idx[k + 1])])
                    phi[k][t] = A + B
                continue
            for k in range(n):
                phi[k][t] = Counter(features[idx[k]:idx[k + 1]])
        return phi

    def _with_phi(self, fn, *args):
        """Run a generic-driver method with `self.X` / `self._Y` holding the per-graph Counters."""
        data = self.X
        self.X = self._phi_X
        try:
            return fn(*args)
        finally:
            self.X = data

    def _metric_fit_transform(self):
        levels = self._device_bins(self.X, None)
        self._hd_cache = [self._fit_ids(b)[0] for b, _ in levels]
        self._phi_X = self._phi(levels, self.X.sizes, 0)
        km = self._with_phi(self._calculate_kernel_matrix)
        self._X_diag = np.diagonal(km)
        if self.normalize:  # kernel.py:196-203
            self._warn_unnormalizable(self._X_diag)
            with np.errstate(invalid="ignore", divide="ignore"):
                return km / np.sqrt(np.outer(self._X_diag, self._X_diag))
        return km

    def _metric_transform(self, Y):
        levels = self._device_bins(self.X, Y)
        hd_fit = [self._fit_ids(b[:int(np.sum(self.X.sizes))])[0] for b, _ in levels]
        self._hd_cache = hd_fit
        self._phi_X = self._phi(levels, self.X.sizes, 0)
        phi_Y = self._phi(levels, Y.sizes, int(np.sum(self.X.sizes)), hd_fit, split=Y.u_full is not None)
        km = self._with_phi(self._calculate_kernel_matrix, phi_Y)
        self._Y = phi_Y
        self._is_transformed = True
        if self.normalize:  # kernel.py:155-164
            X_diag, Y_diag = self._with_phi(self._pairwise_diagonal)
            self._warn_unnormalizable(X_diag, Y_diag)
            with np.errstate(invalid="ignore", divide="ignore"):
                km /= np.sqrt(np.outer(Y_diag, X_diag))
        return km

    # ---- device side
    def _pk_inputs(self, X, Y):
        """(graph sizes, T list, label ids, P0 or None, u [t_max, dim], b, dim, dim_orig, flags) of the joint X || Y run."""
        parts = [X] if Y is None else [X, Y]
        sizes = np.concatenate([p.sizes for p in parts])
        mats = [T for p in parts for T in p.T]
        ids = np.concatenate([p.ids for p in parts])
        dim = parts[-1].dim
        dim_orig = len(self._enum_labels)
        flags = _lib.GK_PK_SQRT if self.take_sqrt_ else 0
        if Y is not None and Y.u_full is not None:
            u = np.stack(Y.u_full)
            flags |= _lib.GK_PK_NEW_LABELS
        else:
            u = np.stack(self._u)
            dim_orig = dim
        return sizes, mats, ids, None, u, np.asarray(self._b, dtype=np.float64), dim, dim_orig, flags

    def _pk_features(self, eng, X, Y):
        """Pack T's pattern and run gk_pk_features on `eng` for the joint X || Y block.  Returns (stats, V, n_graphs,
        n_fit)."""
        sizes, mats, ids, p0, u, b, dim, dim_orig, flags = self._pk_inputs(X, Y)
        gp = np.concatenate([[0], np.cumsum(sizes)])
        rows, cols, vals = [], [], []
        for g, T in enumerate(mats):
            ii, jj = np.nonzero(T)
            rows.append(ii + gp[g]); cols.append(jj + gp[g]); vals.append(T[ii, jj])
        V = int(gp[-1])
        r = np.concatenate(rows).astype(np.int64) if rows else np.zeros(0, np.int64)
        c = np.concatenate(cols).astype(np.int32) if cols else np.zeros(0, np.int32)
        v = np.concatenate(vals).astype(np.float64) if vals else np.zeros(0)
        rp = np.concatenate([[0], np.cumsum(np.bincount(r, minlength=V))])
        n_fit = len(X.sizes)
        eng.pack(gp, rp, c, None if self.attr_ else ids, None, None)
        try:
            st = eng.pk_features(self.t_max, self.w, u, b, dim, dim_orig, n_fit, v, p0, flags)
        except NotImplementedError as e:
            if "NaN" in str(e):  # the reference's hash dictionary cannot look a NaN bin up (propagation.py:282)
                raise KeyError(np.float64(np.nan)) from e
            raise
        return st, V, len(sizes), n_fit

    def _pk_run(self, X, Y, want_matrix=True, device_ptr=None):
        """gk_pk_features -> gk_gram.  Returns (K, xdiag, ydiag)."""
        with _lib.engine(getattr(self, "device_", None)) as eng:
            self.stats_, _, n_graphs, n_fit = self._pk_features(eng, X, Y)
            out = False if not want_matrix else None
            K, xd, yd = eng.gram(n_graphs, n_fit=n_fit, normalize=bool(self.normalize) and want_matrix,
                                 out=out if device_ptr is None else None, device_ptr=device_ptr, stats=self.stats_)
        if self.verbose:
            print(type(self).__name__, self.stats_.as_dict())
        return K, xd, yd


class PropagationAttr(Propagation):
    """Propagation kernel for attributed graphs (propagation.py:426-689).

    P starts as the vertex attributes, in the dtype numpy's vstack gives them, and keeps that dtype: every propagation
    step is rounded to float32, or truncated toward zero for integer attributes, as the reference's assignment into P
    does.  A vertex's bin at level t is the tuple floor((P_v * u_t + b_t) / w) (element-wise, u_t Gaussian or Cauchy for
    M="L1", b_t = w * randn(d)).  Only the plain transform exists, as in the reference.  Deviations as for
    Propagation; attributes of a dtype other than float64, float32 or signed integers, a float32 T over float32
    attributes, and transform attributes of another dtype than the fitted ones raise NotImplementedError."""

    _graph_format = "adjacency"
    attr_ = True

    def __init__(self, n_jobs=None, verbose=False, normalize=False, random_state=None, metric=_pk_dot, M="L1", t_max=5,
                 w=4):
        super().__init__(n_jobs=n_jobs, verbose=verbose, normalize=normalize, random_state=random_state, metric=metric,
                         M=M, t_max=t_max, w=w)

    def initialize(self):
        super().initialize()

    def parse_input(self, X):
        """propagation.py:496-608: attributes, their dimension and the draws."""
        Attr = []
        els = self._elements(X, lambda lab: Attr.append(np.array([lab[j] for j in range(len(lab))])))
        data = Fitted(None, None, {})
        data.T, data.sparse = self._transitions(els)
        try:
            P = np.vstack(Attr)
        except ValueError:
            raise ValueError("Attribute dimensions should be the same, for all graphs")
        if self._method_calling == 1:
            self._dim = P.shape[1]
        elif self._dim != P.shape[1]:
            raise ValueError("transform attribute vectors should have the same dimension as in fit")
        if not els:
            raise ValueError("Parsed input is empty")
        if P.dtype == np.float64:
            data.store = 0
        elif P.dtype == np.float32:
            data.store = _lib.GK_PK_STORE_F32
        elif P.dtype.kind == "i":
            data.store = _lib.GK_PK_STORE_INT
        else:
            raise NotImplementedError("PropagationAttr: attributes of dtype " + str(P.dtype) + " are not supported "
                                      "(float64, float32 or signed integers)")
        if data.store == _lib.GK_PK_STORE_F32 and any(isinstance(T, np.ndarray) and T.dtype == np.float32
                                                      for _, _, T in els):
            raise NotImplementedError("PropagationAttr: a float32 transition matrix over float32 attributes is "
                                      "propagated in float32 by numpy; only float64 propagation runs on the device")
        data.P = P
        data.sizes = np.array([len(lab) for _, lab, _ in els], dtype=np.int64)
        data.ids = None
        data.u_full = None  # no new-label branch for attributes
        if self._method_calling == 1:
            self._u, self._b = list(), list()
            for t in range(self.t_max):
                u = self.random_state_.randn(self._dim)
                if self.take_cauchy_:
                    u = np.divide(u, self.random_state_.randn(self._dim))
                self._u.append(u)
                self._b.append(self.w * self.random_state_.randn(self._dim))
            self._hd_cache = None
        self._sparse_step_error(data)
        return data

    def _pk_inputs(self, X, Y):
        parts = [X] if Y is None else [X, Y]
        if len({p.store for p in parts}) != 1:
            raise NotImplementedError("PropagationAttr: fit and transform attributes of different dtypes")
        sizes = np.concatenate([p.sizes for p in parts])
        mats = [T for p in parts for T in p.T]
        p0 = np.concatenate([np.asarray(p.P, dtype=np.float64) for p in parts])
        return (sizes, mats, None, p0, np.stack(self._u), np.stack(self._b), self._dim, self._dim,
                _lib.GK_PK_ATTR | parts[0].store)


# ------------------------------------------------------------------------------
# The embedding calls of PyramidMatch, by module-level name: `eigs` for graphs of more than d + 1 vertices, `eig` for
# the others, with the reference's arguments.  scipy's eigs draws its start vector from OS entropy unless it is given an
# `rng`, so the reference's K is not reproducible; substituting a seeded `eigs` here (tests) makes both deterministic.
from scipy.sparse import csr_matrix as _csr_matrix  # noqa: E402
from scipy.sparse.linalg import eigs  # noqa: E402

eig = np.linalg.eig

_PM_ELEMENT_MSG = ("each element of X must be either a graph object or a list with at least a graph like object and "
                   "node labels dict \n")


def pm_embedding(A, d):
    """|U| of one graph's adjacency matrix A as pyramid_match.py:135-147 makes it: the d eigenvectors of eigs (n > d + 1)
    or the first d columns of eig, ordered by descending eigenvalue (numpy's argsort, complex for directed graphs)."""
    if A.shape[0] > d + 1:
        Lambda, U = eigs(_csr_matrix(A, dtype=float), k=d, ncv=10 * d)
        U = U[:, Lambda.argsort()[::-1]]
    else:
        Lambda, U = eig(A)
        U = U[:, Lambda.argsort()[::-1]]
        U = U[:, :d]
    return np.absolute(U)


def _pm_empty_error(g, with_labels):
    """The error the reference meets on a graph without vertices (inside Graph or its own unpacking)."""
    if isinstance(g, dict):
        return TypeError("cannot unpack non-iterable NoneType object")
    if isinstance(g, (list, tuple)):
        return IndexError("tuple index out of range")
    if with_labels:
        return ValueError("Graph does not have any labels for vertices.")
    return ValueError("not enough values to unpack (expected 2, got 1)")


class _PmData:
    """Host state of a PyramidMatch input: per embedding set the |U| of every vertex ([S, V, d], zero past a graph's
    column count) and the column counts [S, N]; graph sizes; per-vertex labels (or None)."""

    def __init__(self, sizes, U, n_cols, labels, skip=None):
        self.sizes = np.asarray(sizes, dtype=np.int64)
        self.U = U
        self.n_cols = n_cols
        self.labels = labels
        self.skip = skip  # [V] bool: packed vertices without embedding (outside the base kernel's graph), or None

    def __len__(self):
        return len(self.sizes)

    @staticmethod
    def concat(a, b):
        labels = None if a.labels is None else list(a.labels) + list(b.labels)
        skip = None
        if a.skip is not None or b.skip is not None:
            skip = np.concatenate([np.zeros(a.U.shape[1], bool) if a.skip is None else a.skip,
                                   np.zeros(b.U.shape[1], bool) if b.skip is None else b.skip])
        return _PmData(np.concatenate([a.sizes, b.sizes]), np.concatenate([a.U, b.U], axis=1),
                       np.concatenate([a.n_cols, b.n_cols], axis=1), labels, skip)


def pm_embed_sets(mats, d, n_sets):
    """(U [n_sets, V, d], n_cols [n_sets, N]) of the adjacency matrices `mats`: n_sets embedding passes, set-major
    (WeisfeilerLehman over PyramidMatch fits a fresh kernel per level, each of which embeds every graph again)."""
    sizes = np.array([A.shape[0] for A in mats], dtype=np.int64)
    gp = np.concatenate([[0], np.cumsum(sizes)])
    U = np.zeros((n_sets, int(gp[-1]), d))
    n_cols = np.zeros((n_sets, len(mats)), dtype=np.int32)
    for s in range(n_sets):
        for g, A in enumerate(mats):
            u = pm_embedding(A, d)
            U[s, gp[g]:gp[g + 1], :u.shape[1]] = u
            n_cols[s, g] = u.shape[1]
    return U, n_cols


def pm_check_cells(U, n_cols, sizes, L):
    """The reference's own failures while binning (pyramid_match.py:213-221): int() of a NaN cell, a cell past the
    clamp (u >= 1 + 2^-j) as an index out of range."""
    if L == 0 or U.size == 0:
        return
    gp = np.concatenate([[0], np.cumsum(sizes)])
    mask = np.arange(U.shape[2])[None, None, :] < np.repeat(n_cols, np.diff(gp), axis=1)[:, :, None]
    u = U[mask]
    if np.isnan(u).any():
        raise ValueError("cannot convert float NaN to integer")
    umax = float(u.max()) if u.size else 0.0
    for j in range(L):
        k = 2 ** j
        if np.floor(umax * k) > k:
            raise IndexError("index %d is out of bounds for axis 1 with size %d" % (int(np.floor(umax * k)), k))


class PyramidMatch(Kernel):
    """Pyramid match kernel (pyramid_match.py:18-285; Nikolentzos et al. 2017).

    Every vertex is embedded by the absolute values of d eigenvectors of its graph's adjacency matrix; level j < L
    splits the unit hypercube into 2^j cells per dimension, and K sums the levels' histogram intersections with the
    reference's weights.  The embedding runs on the host with the reference's own scipy / numpy calls (`eigs`, `eig`
    above); the cells, the per-level intersections (an exact integer Gram per level) and the fp64 combine run on the
    device.  Given the same embeddings, K equals the reference's bit for bit, including its combine, whose two
    statements sit inside the level loop (a graph's self similarity at L = 2 is 1.5 times its vertex-dimension count).

    Deviations: L > 64, d * (largest graph) >= 2^24 and V * d >= 2^31 raise NotImplementedError, as does a
    (label, dimension, cell) key that does not fit 64 bits."""

    _graph_format = "adjacency"

    def __init__(self, n_jobs=None, normalize=False, verbose=False, with_labels=True, L=4, d=6):
        super().__init__(n_jobs=n_jobs, normalize=normalize, verbose=verbose)
        self.with_labels = with_labels
        self.L = L
        self.d = d
        self._initialized.update({"d": False, "L": False, "with_labels": False})

    def initialize(self):
        """pyramid_match.py:62-81."""
        super().initialize()
        if not self._initialized["with_labels"]:
            if type(self.with_labels) != bool:
                raise TypeError("with labels must be a boolean variable")
            self._initialized["with_labels"] = True
        if not self._initialized["L"]:
            if type(self.L) is not int or self.L < 0:
                raise TypeError("L: the number of levels must be an integer bigger equal to 0")
            self._initialized["L"] = True
        if not self._initialized["d"]:
            if type(self.d) is not int or self.d < 1:
                raise TypeError("d: hypercube dimension must be an integer bigger than 1")
            self._initialized["d"] = True

    # ---- input
    def _elements(self, X):
        """(adjacency matrix, labels in index order or None) of every element (pyramid_match.py:102-153); the
        embedding calls are made afterwards, in input order."""
        from .packing import adjacency_and_labels
        if isinstance(X, Block):  # datasets.read_tu
            out = _block_adjacency(X, self.with_labels)
            if any(A.shape[0] == 0 for A, _ in out):
                raise ValueError("Graph does not have any labels for vertices." if self.with_labels else
                                 "not enough values to unpack (expected 2, got 1)")
            if not out:
                raise ValueError("parsed input is empty")
            return out
        if not isinstance(X, Iterable):
            raise TypeError("input must be an iterable\n")
        out = []
        for idx, x in enumerate(iter(X)):
            if isinstance(x, Graph):
                x = x.as_element()
            is_iter = isinstance(x, Iterable)
            if is_iter:
                x = list(x)
            if not (is_iter and (len(x) == 0 or (len(x) >= 1 and not self.with_labels) or
                                 (len(x) >= 2 and self.with_labels))):
                raise TypeError(_PM_ELEMENT_MSG)
            if len(x) == 0:
                warnings.warn("Ignoring empty element on index: " + str(idx))
                continue
            if isinstance(x[0], (list, tuple)) and len(x[0]) == 0:
                raise _pm_empty_error(x[0], self.with_labels)
            A, labels = adjacency_and_labels(x[0], x[1] if self.with_labels else None)
            if A.shape[0] == 0:
                raise _pm_empty_error(x[0], self.with_labels)
            out.append((A, labels))
        if not out:
            raise ValueError("parsed input is empty")
        return out

    def parse_input(self, X):
        import time
        els = self._elements(X)
        t0 = time.perf_counter()
        U, n_cols = pm_embed_sets([A for A, _ in els], self.d, 1)
        self.ms_host_embed_ = (time.perf_counter() - t0) * 1e3
        data = _PmData([A.shape[0] for A, _ in els], U, n_cols, None)
        pm_check_cells(U, n_cols, data.sizes, self.L)
        if self.with_labels:
            data.labels = [l for _, L in els for l in L]
            if self._method_calling in (1, 2):  # pyramid_match.py:158-165
                labels = set()
                for _, L in els:
                    labels |= set(L)
                self._num_labels = len(labels)
                self._labels = {l: i for (i, l) in enumerate(labels)}
        return data

    def _label_ids(self, data, n_fit):
        """Packed label ids: the fit enumeration, labels unseen at fit after it (pyramid_match.py:167-174) -- their rows
        never meet a fitted graph's, as the reference's row cut `yp[:xp.shape[0]]` has it."""
        known = dict(self._labels)
        ids = np.empty(len(data.labels), dtype=np.int32)
        for i, l in enumerate(data.labels):
            v = known.get(l)
            if v is None:
                v = known[l] = len(known)
            ids[i] = v
        return ids

    # ---- estimator protocol
    def fit_transform(self, X, y=None):
        self._method_calling = 2
        self.fit(X)
        K, xdiag, _ = self._pm_run(self.X, len(self.X))
        self._X_diag = xdiag
        if self.normalize:
            self._warn_unnormalizable(xdiag)
        return K

    def transform(self, X):
        self._method_calling = 3
        check_is_fitted(self, ["X"])
        if X is None:
            raise ValueError("`transform` input cannot be None")
        Y = self.parse_input(X)
        K, xdiag, ydiag = self._pm_run(_PmData.concat(self.X, Y), len(self.X))
        self._X_diag, self._Y_diag = xdiag, ydiag
        self._is_transformed = True
        if self.normalize:
            self._warn_unnormalizable(xdiag, ydiag)
        return K

    def diagonal(self):
        check_is_fitted(self, ["X"])
        try:
            check_is_fitted(self, ["_X_diag"])
        except NotFittedError:
            _, self._X_diag, _ = self._pm_run(self.X, len(self.X), want_matrix=False)
        if getattr(self, "_is_transformed", False):
            return self._X_diag, self._Y_diag
        return self._X_diag

    def _pm_run(self, data, n_fit, want_matrix=True, device_ptr=None):
        """pack the vertex sets -> gk_pm_features (cells, per-level columns) -> gk_gram (per-level Grams, fp64 combine).
        Returns (K, xdiag, ydiag)."""
        ids = self._label_ids(data, n_fit) if self.with_labels else None
        gp = np.concatenate([[0], np.cumsum(data.sizes)])
        V = int(gp[-1])
        with _lib.engine(getattr(self, "device_", None)) as eng:
            eng.pack(gp, np.zeros(V + 1, dtype=np.int32), np.zeros(0, dtype=np.int32), ids, None, None)
            self.stats_ = eng.pm_features(self.L, self.d, data.U, data.n_cols,
                                          flags=_lib.GK_PM_LABELS if self.with_labels else 0, skip=data.skip)
            out = False if not want_matrix else None
            K, xd, yd = eng.gram(len(data), n_fit=n_fit, normalize=bool(self.normalize) and want_matrix,
                                 out=out if device_ptr is None else None, device_ptr=device_ptr, stats=self.stats_)
        if self.verbose:
            print(type(self).__name__, self.stats_.as_dict())
        return K, xd, yd


# ------------------------------------------------------------------------------
def hc_width(n_labels):
    """Columns of the reference's Hadamard matrix, `2 ** ceil(log2(nl))` (hadamard_code.py:187), in integers."""
    return 1 if n_labels <= 1 else 1 << (int(n_labels) - 1).bit_length()


def hc_edge_keys(g):
    """The keys of the reference's edge dictionary of graph-like `g` (graph.py:1182-1204): None for an adjacency
    input (every vertex is a key), else the endpoints of the listed edges plus the keys of a dict-of-dicts, where
    `{u: {}}` keeps u (graph.py:1660-1667); `{u: []}` does not."""
    from .packing import classify
    kind = classify(g)
    if kind is None:
        raise ValueError("Unsupported input type. For more information check the documentation, concerning valid input "
                         "types for graph type object.")
    if kind == "adjacency":
        return None
    if kind == "dict_tuple":
        return set(chain.from_iterable(g))
    if kind == "dict_list":
        return {u for u, lst in g.items() if lst}.union(chain.from_iterable(g.values()))
    if kind == "dict_dict":
        return set(g).union(chain.from_iterable(g.values()))
    return set(chain.from_iterable((t[0], t[1]) for t in g))


def hc_enumerate(label_dicts, labels_enum=None):
    """The reference's label enumeration (hadamard_code.py:178-181): graph by graph, `for v in set(label.values())`,
    new labels numbered on from the fitted enumeration.  Returns a new dict."""
    enum = {} if labels_enum is None else dict(labels_enum)
    for L in label_dicts:
        for v in set(L.values()):
            if v not in enum:
                enum[v] = len(enum)
    return enum


def _enum_ids(labels, enum):
    """Enumeration id of every packed vertex label."""
    if isinstance(labels, np.ndarray):
        uniq, inv = np.unique(labels, return_inverse=True)
        lut = np.fromiter((enum[int(u)] for u in uniq.tolist()), dtype=np.int32, count=len(uniq))
        return lut[inv.reshape(-1)]
    return np.fromiter((enum[l] for l in labels), dtype=np.int32, count=len(labels))


class HadamardCode(Kernel):
    """Hadamard code kernel (hadamard_code.py:24-391): K = sum over n_iter levels of the base kernel on the vertices'
    Hadamard-code vectors.  Level 0 gives every labelled vertex row `enumeration id` of the W x W Sylvester Hadamard
    matrix (W = 2^ceil(log2 nl)); level i adds every edge-dictionary key's out-neighbour vectors to its own, in int64
    arithmetic that wraps.  The vectors, their exact classes and the per-level base-kernel features are computed on
    the device (gk_hc_features); the host replays the reference's label enumeration, so the device vectors are the
    reference's tuples entry for entry.

    Base kernels: VertexHistogram (default), ShortestPath(with_labels=True), EdgeHistogram, SubgraphMatching (kv
    `_dirac` or None), PyramidMatch and NeighborhoodSubgraphPairwiseDistance.  Labelled vertices that are not keys of
    the edge dictionary count at level 0 only, as in the reference.  SubgraphMatching counts every level's cliques in
    one enumeration over the union of the levels' product graphs, each clique at the levels where all its vertex pairs
    share their classes (DESIGN 4.24); PyramidMatch reads every level's device classes; NSPD hashes the reference's
    label strings, str() of each class's tuple of numpy int64, built on the host from one device vector per class.
    A transform whose new labels widen the Hadamard matrix shares no label with the fitted graphs: K is zero for the
    bases that read labels, as in the reference.  A custom kv and a datasets.read_tu block raise NotImplementedError
    for these three bases."""

    _graph_format = "auto"
    _nan_to_num = True

    def __init__(self, n_jobs=None, verbose=False, normalize=False, n_iter=5, base_graph_kernel=None):
        super().__init__(n_jobs=n_jobs, verbose=verbose, normalize=normalize)
        self.n_iter = n_iter
        self.base_graph_kernel = base_graph_kernel
        self._initialized.update({"n_iter": False, "base_graph_kernel": False})

    def initialize(self):
        if not self._initialized["n_jobs"]:  # kernel.py:386-399: validated, then one device job
            if type(self.n_jobs) is not int and self.n_jobs is not None:
                raise ValueError("n_jobs parameter must be an int indicating the number of jobs as in joblib or None")
            self._parallel = None
            self._initialized["n_jobs"] = True
        if not self._initialized["base_graph_kernel"]:  # hadamard_code.py:68-97
            self.base_graph_kernel_ = parse_base_kernel(
                self, VertexHistogram, (VertexHistogram, ShortestPath, EdgeHistogram, SubgraphMatching, PyramidMatch,
                                        NeighborhoodSubgraphPairwiseDistance),
                "grakel_b200 runs HadamardCode over VertexHistogram, ShortestPath, EdgeHistogram, SubgraphMatching, "
                "PyramidMatch or NeighborhoodSubgraphPairwiseDistance; other base kernels are outside the device hot "
                "path",
                lambda base, params: level_base_check(self, "HadamardCode", base, params, "Hadamard-code tuples",
                                                      "Hadamard codes", "n_iter"))
            self._initialized["base_graph_kernel"] = True
        if not self._initialized["n_iter"]:  # :99-102
            if type(self.n_iter) is not int or self.n_iter <= 0:
                raise TypeError("'n_iter' must be a positive integer")
            self._initialized["n_iter"] = True

    # ---- host parsing -----------------------------------------------------------
    def _elements(self, X):
        """[graph, labels] or [graph, labels, edge labels] per kept element, with the reference's element checks
        (hadamard_code.py:142-176)."""
        if not isinstance(X, Iterable):
            raise TypeError("input must be an iterable\n")
        out = []
        for idx, x in enumerate(iter(X)):
            is_iter = False
            if isinstance(x, Iterable):
                x, is_iter = list(x), True
            if is_iter and (len(x) == 0 or len(x) >= 2):
                if len(x) == 0:
                    warnings.warn("Ignoring empty element on index: " + str(idx))
                    continue
                out.append(x[:3])
            elif type(x) is Graph:
                if self.base_graph_kernel_[0] in _HC_GRAPH_BASES:
                    # the reference asks a Graph for its edge labels with purpose "auto" (hadamard_code.py:163)
                    raise ValueError("unsupported label purpose")
                el = x.as_element()
                out.append(el if x.edge_labels else el[:2])
            else:
                raise TypeError("each element of X must be either a graph object or a list with at least a graph like "
                                "object and node labels dict \n")
        if not out:
            raise ValueError("parsed input is empty")
        return out

    def _parse(self, X, labels_enum):
        """(Fitted, extended enumeration) of one input."""
        base = self.base_graph_kernel_[0]
        if isinstance(X, Block):  # packed input (datasets.read_tu): integer labels
            if base is EdgeHistogram:
                raise NotImplementedError("packed blocks carry no edge-label entries; pass the list of graphs")
            if base in _HC_GRAPH_BASES:
                raise NotImplementedError("HadamardCode over %s needs every graph's edge dictionary and edge labels "
                                          "(its adjacency matrix for PyramidMatch); pass the list of graphs"
                                          % base.__name__)
            block = X.require("wl", "sp")
            gp = np.asarray(block.graph_ptr)
            labels = np.asarray(block.labels)
            enum = {} if labels_enum is None else dict(labels_enum)
            for g in range(block.n_graphs):
                for v in set(labels[gp[g]:gp[g + 1]].tolist()):
                    if v not in enum:
                        enum[v] = len(enum)
            skip = None
            if block.mode == "wl" and self.n_iter > 1:  # the edge-dictionary keys are the endpoints of the edges
                rp = np.asarray(block.row_ptr)
                key = np.diff(rp) > 0
                key[np.asarray(block.col_idx)] = True
                skip = None if key.all() else ~key
            elif block.mode == "sp" and base is not ShortestPath:
                raise ValueError("this block was packed for another kernel (vertex set 'sp', needed 'wl'): see "
                                 "grakel_b200.datasets.read_tu(kernel=...)")
            return Fitted(block, _enum_ids(labels, enum), skip=skip), enum
        els = self._elements(X)
        enum = hc_enumerate((x[1] for x in els), labels_enum)
        if base is EdgeHistogram:
            values = _edge_label_values(els)
            sizes = np.concatenate([[0], np.cumsum([len(v) for v in values])])
            block = Block(sizes, np.zeros(int(sizes[-1]) + 1, dtype=np.int64), np.zeros(0, dtype=np.int64), None,
                          [l for v in values for l in v])
            return Fitted(block, None), enum
        if base is ShortestPath:
            # the base kernel receives every element's own graph object (hadamard_code.py:175, 197): its vertices, and
            # Floyd-Warshall or Dijkstra path sums as the element's format implies (_path_sum_order).  Its vertices
            # outside the edge dictionary's keys have no edge, so their labels never reach a path feature.
            block = pack([x[:2] for x in els], "sp", want_weights=True,
                         fw_zero_is_absent=self.base_graph_kernel_[1].get("algorithm_type") == "floyd_warshall",
                         type_error_msg="each element of X must have at least one and at most 3 elements\n")
            return Fitted(block, _enum_ids(block.labels, enum)), enum
        if self.n_iter == 1 and base not in _HC_GRAPH_BASES:  # level 0 only: the label multisets
            labels = [l for x in els for l in x[1].values()]
            sizes = np.concatenate([[0], np.cumsum([len(x[1]) for x in els])])
            block = Block(sizes, np.zeros(int(sizes[-1]) + 1, dtype=np.int64), np.zeros(0, dtype=np.int64), None, labels)
            return Fitted(block, _enum_ids(labels, enum)), enum
        # packed vertices: the keys of every labels dictionary, in its order ('wl' packing)
        skip = []
        for x in els:
            keys = hc_edge_keys(x[0])
            if keys is None:
                skip.append(np.zeros(len(x[1]), dtype=bool))
                continue
            missing = keys.difference(x[1])
            if missing:  # the reference's old_label[k] (hadamard_code.py:209)
                raise KeyError(next(iter(missing)))
            skip.append(np.fromiter((k not in keys for k in x[1]), dtype=bool, count=len(x[1])))
        skip = np.concatenate(skip)
        block = pack([x[:2] for x in els], "wl", len_ok=lambda n: n >= 2)
        data = Fitted(block, _enum_ids(block.labels, enum), skip=skip if skip.any() else None)
        if base is PyramidMatch:
            p = self.base_graph_kernel_[1]
            data.pm, self.ms_host_embed_ = pm_level_embeddings(els, block, p.get("d", 6), p.get("L", 4), self.n_iter,
                                                               "HadamardCode")
        elif base in _HC_GRAPH_BASES:
            data.base = base_graph_data(els, block, base, self._sm, "HadamardCode")
        return data, enum

    def _eh_ids(self, data, known):
        ids, new = label_ids(data.block.labels, known, sort_new=False)
        data.ids = ids
        return new

    # ---- estimator protocol -----------------------------------------------------
    def fit(self, X, y=None):
        self._is_transformed = False
        self._method_calling = 1
        self.initialize()
        if X is None:
            raise ValueError("`fit` input cannot be None")
        self._fit(X)
        return self

    def _fit(self, X):
        if hasattr(self, "_X_diag"):
            delattr(self, "_X_diag")
        data, enum = self._parse(X, None)
        if self.base_graph_kernel_[0] is EdgeHistogram:
            self._eh_labels = self._eh_ids(data, None)
            self._width = hc_width(len(self._eh_labels))
        else:
            self._width = hc_width(len(enum))
        self.X = data
        self._labels_enum = enum

    def fit_transform(self, X, y=None):
        self._method_calling = 2
        self._is_transformed = False
        self.initialize()
        if X is None:
            raise ValueError("transform input cannot be None")
        self._fit(X)
        K, xdiag, _ = self._run(self.X, len(self.X), self._width)
        self._X_diag = xdiag
        return K

    def transform(self, X):
        self._method_calling = 3
        check_is_fitted(self, ["X"])
        if X is None:
            raise ValueError("transform input cannot be None")
        Y, enum = self._parse(X, self._labels_enum)
        n_x, n_y = len(self.X), len(Y)
        if self.base_graph_kernel_[0] is EdgeHistogram:
            new = self._eh_ids(Y, self._eh_labels)
            width = hc_width(len(self._eh_labels) + len(new))
        else:
            width = hc_width(len(enum))
        if width == self._width or self.base_graph_kernel_[0] is EdgeHistogram or not self._reads_labels():
            K, xdiag, ydiag = self._run(Fitted.concat(self.X, Y), n_x, width)
        else:
            # the vectors of Y are longer than every fitted vector: no label is shared (hadamard_code.py:187, 235) and
            # every Y graph is only similar to itself, at its own width.  (NSPD: the label strings str(tuple) of Y are
            # longer than every fitted one, so no neighbourhood hash is shared either.)
            _, ydiag, _ = self._run(Y, n_y, width, want_matrix=False)
            try:
                check_is_fitted(self, ["_X_diag"])
                xdiag = self._X_diag
            except NotFittedError:
                _, xdiag, _ = self._run(self.X, n_x, self._width, want_matrix=False)
            K = np.zeros((n_y, n_x))
        self._X_diag = xdiag
        self._Y_diag = ydiag
        self._is_transformed = True
        return K

    def diagonal(self):
        check_is_fitted(self, ["X"])
        try:
            check_is_fitted(self, ["_X_diag"])
        except NotFittedError:
            _, self._X_diag, _ = self._run(self.X, len(self.X), self._width, want_matrix=False)
        if getattr(self, "_is_transformed", False):
            return self._X_diag, self._Y_diag
        return self._X_diag

    # ---- device -----------------------------------------------------------------
    def _dijkstra_order(self, block):
        return _path_sum_order(block, self.base_graph_kernel_[1].get("algorithm_type", "auto"))

    def _reads_labels(self):
        """Whether the base kernel reads the Hadamard codes: not SubgraphMatching(kv=None), not
        PyramidMatch(with_labels=False)."""
        base, p = self.base_graph_kernel_
        if base is SubgraphMatching:
            return self._sm.kv is not None
        if base is PyramidMatch:
            return bool(p.get("with_labels", True))
        return True

    def _run(self, data, n_fit, width, want_matrix=True, row_range=None, device_ptr=None):
        """pack -> gk_hc_features -> gk_gram.  Returns (K, xdiag, ydiag)."""
        block = data.block
        base = self.base_graph_kernel_[0]
        if base in _HC_GRAPH_BASES:
            return self._base_run(data, n_fit, width, want_matrix, row_range, device_ptr)
        with _lib.engine(getattr(self, "device_", None)) as eng:
            eng.pack(block.graph_ptr, block.row_ptr, block.col_idx, data.ids,
                     block.weights if base is ShortestPath else None, None)
            if base is ShortestPath:
                self.stats_ = eng.hc_features(self.n_iter, width, sp=True, dijkstra_order=self._dijkstra_order(block))
            else:
                self.stats_ = eng.hc_features(self.n_iter, width, skip=data.skip)
            K, xd, yd = eng.gram(block.n_graphs, n_fit=n_fit, normalize=bool(self.normalize) and want_matrix,
                                 nan_to_num=True, out=None if want_matrix else False, stats=self.stats_)
        if self.verbose:
            print(type(self).__name__, self.stats_.as_dict())
        return K, xd, yd

    def _relabel(self, eng, data, width):
        """Pack the HadamardCode vertex set and relabel it on the device: every level's classes stay on `eng`
        (gk_hc_features)."""
        block = data.block
        eng.pack(block.graph_ptr, block.row_ptr, block.col_idx, data.ids, None, None)
        eng.hc_features(self.n_iter, width, skip=data.skip)

    def _level_classes(self, eng, data, width, vectors=False):
        """The HadamardCode class of every packed vertex at every level, [V, n_iter] (gk_wl_labels: exact vector
        classes, numbered on the device); with `vectors` also, per level, the [V, W] vectors."""
        self._relabel(eng, data, width)
        n_v = data.block.n_vertices
        cls = np.stack([eng.wl_labels(lv, n_v) for lv in range(self.n_iter)], axis=1)
        if not vectors:
            return cls, None
        return cls, [eng.hc_vectors(lv, n_v, width) for lv in range(self.n_iter)]

    def _base_run(self, data, n_fit, width, want_matrix, row_range, device_ptr):
        """HadamardCode over SubgraphMatching, PyramidMatch or NSPD: K = sum over the n_iter levels of the base kernel
        on the level's Hadamard codes, added in level order (hadamard_code.py:217-236, np.sum(axis=0)), by that base's
        level route; DESIGN 4.24."""
        base, p = self.base_graph_kernel_
        reads = self._reads_labels()
        if base is PyramidMatch:
            relabel = functools.partial(self._relabel, data=data, width=width) if reads else None
            return pm_level_run(self, data.pm, data.block, relabel, self.n_iter, p.get("L", 4), p.get("d", 6), n_fit,
                                want_matrix, row_range, device_ptr)
        if base is SubgraphMatching:
            kk = max(1, min(max(int(self._sm.k), 1), max(g[0] for g in data.base.graphs)))
            if self.n_iter * kk > 64:  # gk_sm_hc_features' bin cap, before the relabelling runs
                raise NotImplementedError("HadamardCode over SubgraphMatching: n_iter * min(k, largest graph) is more "
                                          "than 64")
            classes = None
            if reads:
                with _lib.engine(getattr(self, "device_", None)) as eng:
                    classes = self._level_classes(eng, data, width)[0]
            return sm_level_run(self, data.base, classes, False, self.n_iter, n_fit, want_matrix, row_range,
                                device_ptr)
        with _lib.engine(getattr(self, "device_", None)) as eng:
            cls, vecs = self._level_classes(eng, data, width, vectors=True)
        src = data.base.src

        def levels():
            # the reference hashes str(D) + "," + str(label), label the tuple of numpy int64 of the level's vector
            # (neighborhood_subgraph_pairwise_distance.py:443): one string per class, from one vector
            for lv in range(self.n_iter):
                uniq, first, inv = np.unique(cls[src, lv], return_index=True, return_inverse=True)
                rows = vecs[lv][src[first]]
                yield inv.reshape(-1), [str(tuple(row)) for row in rows]
        return nspd_level_sum(self, data.base, levels(), self.n_iter, n_fit, want_matrix, row_range, p.get("r", 3),
                              p.get("d", 4))

    def hc_vectors(self, X, level):
        """[V, W] int64 Hadamard-code vectors of every packed vertex of X at `level` (zeros where a vertex is absent
        from the level), as the fitted estimator's relabelling computes them; rows follow each labels dictionary's
        key order."""
        check_is_fitted(self, ["X"])
        data, enum = self._parse(X, self._labels_enum)
        width = hc_width(len(enum))
        with _lib.engine(getattr(self, "device_", None)) as eng:
            self._relabel(eng, data, width)
            return eng.hc_vectors(level, data.block.n_vertices, width)


# ------------------------------------------------------------------------------
_NSPD_ELEMENT_MSG = ("each element of X must have either a graph with labels for node and edge or 3 elements "
                     "consisting of a graph type object, labels for vertices and labels for edges.")


def _nspd_graph(g, node_labels, edge_labels, with_order=False):
    """One graph as the reference sees it after change_format("adjacency") then ("dictionary") (graph.py:912-1053):
    the spelling is read by packing.classify (graph.py's is_adjacency / is_edge_dictionary), the vertices are the
    indices 0 .. n-1 of an adjacency matrix or of the sorted symbols of an edge dictionary, and an edge survives when
    its adjacency entry is > 0.  Missing vertex or edge labels raise get_labels' ValueError (graph.py:750-770).
    Returns (n, sorted (i, j) edge list, vertex label strings, edge label strings)."""
    if not node_labels:
        raise ValueError("Graph does not have any labels for vertices.")
    if not edge_labels:
        raise ValueError("Graph does not have any labels for edges.")
    A, order = adjacency_and_order(g)
    order = list(order)
    ii, jj = np.nonzero(A > 0)
    edges = sorted(zip(ii.tolist(), jj.tolist()))
    vl = [str(node_labels[s]) for s in order]
    el = [str(edge_labels[(order[i], order[j])]) for i, j in edges]
    if with_order:
        return len(order), edges, vl, el, order
    return len(order), edges, vl, el


class _NspdTokens:
    """str(delta) + "," + str(label) for every delta <= d and label string, ranked by Python's string order, with
    UTF-8 bytes and code-point lengths; the same for the edge label strings."""

    def __init__(self, d, labels, elabels):
        self.n_labels = len(labels)
        toks = [str(t) + "," + s for t in range(d + 1) for s in labels]
        uniq = sorted(set(toks))
        rank = {s: i for i, s in enumerate(uniq)}
        self.tok_rank = np.array([rank[s] for s in toks] or [0], dtype=np.int32)  # padded: never a null pointer
        self.rank_off, self.rank_bytes, self.rank_cp = self._strings(uniq)
        self.el_off, self.el_bytes, self.el_cp = self._strings(elabels)

        self.n_ranks = len(uniq)
        self.n_elabels = len(elabels)

    @staticmethod
    def _strings(strs):
        """(offsets [n + 1], UTF-8 bytes, code points [n]); the byte and code-point arrays are padded by one entry so
        that no pointer is null when n = 0 (the counts passed on are n_ranks / n_elabels, never the padded lengths)."""
        bs = [s.encode("utf-8") for s in strs]
        off = np.zeros(len(bs) + 1, dtype=np.int64)
        off[1:] = np.cumsum([len(b) for b in bs]) if bs else []
        data = np.frombuffer(b"".join(bs) + b"\0", dtype=np.uint8).copy()
        return off, data, np.array([len(s) for s in strs] + [0], dtype=np.int32)


class NeighborhoodSubgraphPairwiseDistance(Kernel):
    """Neighborhood subgraph pairwise distance kernel (neighborhood_subgraph_pairwise_distance.py; Costa & De Grave
    2010).  For every radius rho <= r and distance delta <= d, the pairs of vertices at distance delta are counted by
    the pair of hashes of their radius-rho neighbourhood subgraphs; K is the sum over the levels (rho, delta) of the
    cosine-normalised level Grams.  The BFS levels, the hashes (CPython's set order of the sub-edge sets emulated on
    the device, the APHash of each encoding streamed from sorted token ranks), the per-level columns, the exact
    integer Gram of every level and the reference's fp64 fold run on the device; K equals the reference's bit for
    bit.

    As in the reference, the neighbourhood of level l has BFS radius 2^(l - 1) (produce_neighborhoods unites the
    level-l balls of the level-l ball), `diagonal()` is the number of levels and the vertices are the indices of the
    sorted symbols.  Deviations: (r + 1)(d + 1) > 64 levels raise NotImplementedError, as do a datasets.read_tu
    block (it carries no edge labels) and r > 0 with a graph of 65 535 or more vertices."""

    _graph_format = "dictionary"

    def __init__(self, n_jobs=None, normalize=False, verbose=False, r=3, d=4):
        super().__init__(n_jobs=n_jobs, normalize=normalize, verbose=verbose)
        self.r = r
        self.d = d
        self._initialized.update({"r": False, "d": False})

    def initialize(self):
        if not self._initialized["n_jobs"]:
            if self.n_jobs is not None:
                warnings.warn("no implemented parallelization for NeighborhoodSubgraphPairwiseDistance")
            self._initialized["n_jobs"] = True
        if not self._initialized["r"]:
            if type(self.r) is not int or self.r < 0:
                raise ValueError("r must be a positive integer")
            self._initialized["r"] = True
        if not self._initialized["d"]:
            if type(self.d) is not int or self.d < 0:
                raise ValueError("d must be a positive integer")
            self._initialized["d"] = True
        if (self.r + 1) * (self.d + 1) > 64:
            raise NotImplementedError("NeighborhoodSubgraphPairwiseDistance: at most (r + 1)(d + 1) = 64 levels are "
                                      "supported")

    def parse_input(self, X):
        """The graphs of X as (n, edges, vertex label strings, edge label strings), with the reference's element
        checks."""
        if isinstance(X, Block):
            raise NotImplementedError("packed blocks carry no edge-label entries; pass the list of graphs")
        if not isinstance(X, Iterable):
            raise TypeError("input must be an iterable\n")
        out = []
        for idx, x in enumerate(iter(X)):
            if isinstance(x, Graph):
                x = x.as_element()  # labels it lacks are {}: _nspd_graph raises get_labels' error
            elif isinstance(x, Iterable):
                x = list(x)
                if len(x) == 0:
                    warnings.warn("Ignoring empty element on index: " + str(idx))
                    continue
                if len(x) != 3:
                    raise TypeError(_NSPD_ELEMENT_MSG)
            else:
                raise TypeError(_NSPD_ELEMENT_MSG)
            out.append(_nspd_graph(x[0], x[1], x[2]))
        if not out:
            raise ValueError("parsed input is empty")
        return out

    def fit(self, X, y=None):
        self._method_calling = 1
        self._is_transformed = False
        self.initialize()
        if X is None:
            raise ValueError("`fit` input cannot be None")
        self.X = self.parse_input(X)
        for a in ("_X_diag", "_Y", "_ngy"):
            self.__dict__.pop(a, None)
        self._ngx = len(self.X)
        return self

    def fit_transform(self, X, y=None):
        self._method_calling = 2
        self.fit(X)
        K, xd, _ = self._nspd_run(self.X, len(self.X))
        self._X_diag = xd
        return K

    def transform(self, X, y=None):
        self._method_calling = 3
        check_is_fitted(self, ["X"])
        if X is None:
            raise ValueError("transform input cannot be None")
        Y = self.parse_input(X)
        K, xd, yd = self._nspd_run(self.X + Y, len(self.X))
        self._X_diag, self._Y_diag = xd, yd
        self._ngy = len(Y)
        self._Y = True
        self._is_transformed = True
        return K

    def diagonal(self):
        """The number of levels of each side (the reference's constant self similarity)."""
        check_is_fitted(self, ["X"])
        if getattr(self, "_X_diag", None) is None:
            self._nspd_run(self.X, len(self.X), want_matrix=False)
        if getattr(self, "_is_transformed", False):
            return self._X_diag, self._Y_diag
        return self._X_diag

    def _pack(self, graphs):
        gp, rp, ci, lab, el, sh = [0], [0], [], [], [], []
        lstr, estr = {}, {}
        for n, edges, vl, elab in graphs:
            v0 = gp[-1]
            deg = np.zeros(n, dtype=np.int64)
            for (i, j), s in zip(edges, elab):
                deg[i] += 1
                ci.append(v0 + j)
                el.append(estr.setdefault(s, len(estr)))
            rp.extend((rp[-1] + np.cumsum(deg)).tolist())
            lab.extend(lstr.setdefault(s, len(lstr)) for s in vl)
            sh.extend(hash(i) for i in range(n))
            gp.append(v0 + n)
        tokens = _NspdTokens(self.d, list(lstr), list(estr))
        return (np.array(gp), np.array(rp), np.array(ci, dtype=np.int64), np.array(lab, dtype=np.int64),
                np.array(el, dtype=np.int64), np.array(sh, dtype=np.int64), tokens)

    def _nspd_run(self, graphs, n_fit, want_matrix=True, device_ptr=None, row_range=None, simt=False):
        if self.r > 0 and max(g[0] for g in graphs) >= 65535:  # the device refuses it too; do not pack it first
            raise NotImplementedError("NeighborhoodSubgraphPairwiseDistance: r > 0 with a graph of 65535 or more "
                                      "vertices")
        gp, rp, ci, lab, el, sh, tokens = self._pack(graphs)
        with _lib.engine(getattr(self, "device_", None)) as eng:
            eng.pack(gp, rp, ci, lab, None, None)
            self.stats_, self.delta_mask_ = eng.nspd_features(self.r, self.d, sh, el, tokens)
            K, xd, yd = eng.gram(len(graphs), n_fit=n_fit, normalize=self.normalize, stats=self.stats_,
                                 out=None if want_matrix else False, device_ptr=device_ptr, row_range=row_range,
                                 simt=simt)
        self._X_diag = xd
        if self.verbose:
            print(type(self).__name__, self.stats_.as_dict())
        return K, xd, yd


# ------------------------------------------------------------------------------
def _dirac(a, b):
    """The reference's default vertex and edge kernel, int(a == b).  SubgraphMatching recognises this function by
    identity and compares label ids on the device."""
    return int(a == b)


_SM_ELEMENT_MSG = ("each element of X must be either a graph object or a list with at least a graph like object and "
                   "node, edge labels dict \n")
_SM_TABLE_MAX = 4096
_MISSING = object()


class SubgraphMatching(Kernel):
    """Subgraph matching kernel (subgraph_matching.py; Kriege & Mutzel 2012).  k(x, y) = sum_s lambda_s tv_s, where
    tv[s - 1] sums prod cv * prod |ce| over the vertex sets of size s <= k of the weighted product graph that are
    cliques (every pair has ce != 0) connected by its c-edges (ce > 0).  The clique enumeration of every pair runs on
    the device, one warp per pair, without building the product graph; integer-valued weights (the default `_dirac`,
    None, integer tables) are counted exactly, and the lambdas are folded in np.dot's order, so K equals the
    reference's bit for bit for them.

    Vertices are the indices of an adjacency matrix or the sorted symbols of an edge dictionary, and an edge is an
    adjacency entry > 0, as after the reference's change_format("adjacency").  Deviations: a `kv` / `ke` other than
    `_dirac` or None is called once per pair of distinct labels (the reference calls it once per vertex or edge pair),
    and more than 64 distinct labels on either side raise NotImplementedError; an edge without a label raises the
    reference's TypeError at parse time even when no pair would read it; real lambdas with k + 1 > 15, k < 0 and
    cliques of more than 32 vertices raise NotImplementedError; a count of 2^53 or more raises an error."""

    _graph_format = "all"

    def __init__(self, n_jobs=None, verbose=False, normalize=False, k=5, kv=_dirac, ke=_dirac, lw="uniform"):
        super().__init__(n_jobs=n_jobs, normalize=normalize, verbose=verbose)
        self.k = k
        self.kv = kv
        self.ke = ke
        self.lw = lw
        self._initialized.update({"k": False, "kv": False, "ke": False, "lw": False})

    def initialize(self):
        """subgraph_matching.py:70-120, in its order and with its checks (`k` is validated with `and`)."""
        super().initialize()
        if not self._initialized["k"]:
            if type(self.k) is not int and self.k < 1:
                raise TypeError("k must be an integer greater-equal than 1")
            self._initialized["k"] = True
        if not self._initialized["kv"]:
            if not callable(self.kv) and self.kv is not None:
                raise TypeError("kv must be callable or None")
            self._initialized["kv"] = True
        if not self._initialized["ke"]:
            if not callable(self.ke) and self.ke is not None:
                raise TypeError("ke must be callable or None")
            self._initialized["ke"] = True
        if not self._initialized["lw"]:
            k = self.k + 1
            not_str_iter = type(self.lw) is not str and isinstance(self.lw, Iterable)
            if not_str_iter:
                lw = list(self.lw)
            if not_str_iter and len(lw) == self.k and all(isinstance(x, Real) for x in lw):
                self.lambdas_ = np.array(lw).reshape((1, k))
            elif self.lw == "uniform":
                self.lambdas_ = np.full((1, k), 1.0)
            elif self.lw == "increasing":
                self.lambdas_ = np.arange(1.0, float(k) + 1.0).reshape(1, k)
            elif self.lw == "decreasing":
                self.lambdas_ = np.full((1, k), 1.0) / np.arange(1.0, float(k) + 1.0).reshape(1, k)
            elif self.lw == "strong_decreasing":
                self.lambdas_ = np.full((1, k), 1.0) / np.square(np.arange(1.0, float(k) + 1.0)).reshape(1, k)
            elif callable(self.lw):
                try:
                    self.lambdas_ = np.array([self.lw(i) for i in range(k)]).reshape((1, k))
                except Exception as e:
                    raise TypeError("Incorrect Callable: " + str(e))
            else:
                raise TypeError('lw can either be str with values "uniform", "increasing", "decreasing", '
                                '"strong_decreasing" or an iterable of k+1 elements or a callable of one integer '
                                "argument.")
            self._initialized["lw"] = True
        if int(self.k) < 0:
            raise NotImplementedError("SubgraphMatching: k < 0 has no defined result")

    # ---- input
    def _graph(self, g, node_labels, edge_labels, need_v=None):
        """(n, sorted (i, j) edges without self-loops, vertex labels or None, edge labels or None).  `need_v=False`
        skips the vertex labels (WeisfeilerLehman hands its own)."""
        need_v, need_e = self.kv is not None if need_v is None else need_v, self.ke is not None
        if need_v and not node_labels:
            raise ValueError("Graph does not have any labels for vertices.")
        if need_e and not edge_labels:
            raise ValueError("Graph does not have any labels for edges.")
        A, order = adjacency_and_order(g)
        order = list(order)
        ii, jj = np.nonzero(A > 0)
        edges = [(i, j) for i, j in zip(ii.tolist(), jj.tolist()) if i != j]
        vl = [node_labels[s] for s in order] if need_v else None
        el = None
        if need_e:
            el = []
            for i, j in edges:
                lab = edge_labels.get((order[i], order[j]), _MISSING)
                if lab is _MISSING:
                    # the reference adds a str to the KeyError it catches, which raises a TypeError
                    raise TypeError("unsupported operand type(s) for +: 'KeyError' and 'str'")
                el.append(lab)
        return len(order), edges, vl, el

    def _block(self, X, edge_labels):
        """The graphs of a datasets.read_tu block (the nodes that occur in an edge, as in its edge dictionaries),
        with the block's per-edge label ids `edge_labels` (read_tu's `edge_labels`) when ke is not None."""
        X.require("sp", "core", labels=self.kv is not None)
        if self.ke is not None and edge_labels is None:
            raise ValueError("Graph does not have any labels for edges.")
        gp, rp, ci = X.graph_ptr, X.row_ptr, X.col_idx
        out = []
        for g in range(X.n_graphs):
            a, b = int(gp[g]), int(gp[g + 1])
            ed = {}
            for u in range(a, b):
                for e in range(int(rp[u]), int(rp[u + 1])):
                    v = int(ci[e])
                    if v != u and (X.weights is None or X.weights[e] > 0):
                        ed[(u - a, v - a)] = None if edge_labels is None else int(edge_labels[e])
            edges = sorted(ed)
            out.append((b - a, edges, list(X.labels[a:b]) if self.kv is not None else None,
                        [ed[e] for e in edges] if self.ke is not None else None))
        return out

    def parse_input(self, X):
        """subgraph_matching.py:142-207: Graph objects or 3-element iterables; empty elements are skipped with a
        warning.  Also the result of datasets.read_tu(kernel="SP") (its block and edge labels), or its block alone
        with ke=None."""
        if isinstance(X, dict) and isinstance(X.get("data"), Block):
            return self._block(X["data"], X.get("edge_labels"))
        if isinstance(X, Block):
            if self.ke is not None:
                raise NotImplementedError("a packed block carries no edge labels: pass ke=None or the whole result of "
                                          "datasets.read_tu")
            return self._block(X, None)
        if not isinstance(X, Iterable):
            raise TypeError("input must be an iterable\n")
        out = []
        for idx, x in enumerate(iter(X)):
            if isinstance(x, Graph):
                x = x.as_element()
            elif isinstance(x, Iterable):
                x = list(x)
                if len(x) not in (0, 3):
                    raise TypeError(_SM_ELEMENT_MSG)
                if len(x) == 0:
                    warnings.warn("Ignoring empty element on index: " + str(idx))
                    continue
            else:
                raise TypeError(_SM_ELEMENT_MSG)
            out.append(self._graph(x[0], x[1], x[2]))
        if not out:
            raise ValueError("parsed input is empty")
        return out

    # ---- estimator protocol
    def fit(self, X, y=None):
        self._method_calling = 1
        self._is_transformed = False
        self.initialize()
        if X is None:
            raise ValueError("`fit` input cannot be None")
        self.X = self.parse_input(X)
        self.__dict__.pop("_X_diag", None)
        return self

    def fit_transform(self, X, y=None):
        self._method_calling = 2
        self.fit(X)
        K, xd, _ = self._sm_run(self.X, len(self.X))
        self._X_diag = xd
        if self.normalize:
            self._warn_unnormalizable(xd)
        return K

    def transform(self, X):
        self._method_calling = 3
        check_is_fitted(self, ["X"])
        if X is None:
            raise ValueError("`transform` input cannot be None")
        Y = self.parse_input(X)
        K, xd, yd = self._sm_run(self.X + Y, len(self.X))
        self._X_diag, self._Y_diag = xd, yd
        self._is_transformed = True
        if self.normalize:
            self._warn_unnormalizable(xd, yd)
        return K

    def diagonal(self):
        check_is_fitted(self, ["X"])
        try:
            check_is_fitted(self, ["_X_diag"])
        except NotFittedError:
            _, self._X_diag, _ = self._sm_run(self.X, len(self.X), want_matrix=False)
        if getattr(self, "_is_transformed", False):
            return self._X_diag, self._Y_diag
        return self._X_diag

    @staticmethod
    def _table(fn, labels, what):
        if len(labels) ** 2 > _SM_TABLE_MAX:
            raise NotImplementedError("SubgraphMatching: a custom " + what + " kernel is tabulated over the distinct "
                                      "labels, at most 64 of them (got " + str(len(labels)) + ")")
        return np.array([[float(fn(a, b)) for b in labels] for a in labels], dtype=np.float64).reshape(
            len(labels), len(labels))

    def _pack(self, graphs):
        """(graph_ptr, row_ptr, col_idx, vertex label ids, edge label ids, kv table, ke table, flags)."""
        gp, rp, ci, lab, el = [0], [0], [], [], []
        lid, eid = {}, {}
        for n, edges, vl, elab in graphs:
            v0 = gp[-1]
            deg = np.zeros(n, dtype=np.int64)
            for i, j in edges:
                deg[i] += 1
                ci.append(v0 + j)
            if elab is not None:
                el.extend(eid.setdefault(s, len(eid)) for s in elab)
            rp.extend((rp[-1] + np.cumsum(deg)).tolist())
            if vl is not None:
                lab.extend(lid.setdefault(s, len(lid)) for s in vl)
            gp.append(v0 + n)
        flags, vt, et = 0, None, None
        if self.kv is None:
            flags |= _lib.GK_SM_KV_NONE
        elif self.kv is _dirac:
            flags |= _lib.GK_SM_KV_DIRAC
        else:
            vt = self._table(self.kv, list(lid), "vertex")
        if self.ke is None:
            flags |= _lib.GK_SM_KE_NONE
        elif self.ke is _dirac:
            flags |= _lib.GK_SM_KE_DIRAC
        else:
            et = self._table(self.ke, list(eid), "edge")
        ids = np.array(lab, dtype=np.int64) if self.kv is not None else None
        elids = np.array(el, dtype=np.int64) if self.ke is not None else None
        return (np.array(gp), np.array(rp), np.array(ci, dtype=np.int64), ids, elids, vt, et, flags)

    def _sm_run(self, graphs, n_fit, want_matrix=True, device_ptr=None, row_range=None):
        gp, rp, ci, ids, elids, vt, et, flags = self._pack(graphs)
        with _run_engine(self) as eng:
            eng.pack(gp, rp, ci, ids, None, None)
            self.stats_ = eng.sm_features(int(self.k), self.lambdas_, vt, et, elids, flags)
            K, xd, yd = _gram_or_fold(self, eng, len(graphs), n_fit, want_matrix,
                                      normalize=bool(self.normalize) and want_matrix, device_ptr=device_ptr,
                                      row_range=row_range, stats=self.stats_)
        if self.verbose:
            print(type(self).__name__, self.stats_.as_dict())
        return K, xd, yd


# ------------------------------------------------------------------------------
_ODD_ELEMENT_MSG = ("each element of X must have either a graph with labels for node and edge or 3 elements consisting "
                    "of a graph type object, labels for vertices and labels for edges.")


def _value_ranks(values):
    """Dense ranks of `values` by Python's `<` (equal values share a rank): the order the reference's stable
    `q.sort(key=label)` puts them in."""
    uniq = sorted(set(values))
    at = {}
    r = -1
    for i, v in enumerate(uniq):
        if i == 0 or uniq[i - 1] < v:
            r += 1
        at[v] = r
    return [at[v] for v in values]


def odd_label_tables(labels, graph_ptr):
    """(label id of every vertex: one per distinct str(label), in first-seen order; rank of its value within its
    graph; the distinct strings).  A label whose str has '(', ',' or ')' raises NotImplementedError: the reference's
    identity strings could then be equal for different trees.  Labels of one graph that cannot be compared raise
    TypeError."""
    strs = [str(l) for l in labels]
    ids_of = {}
    ids = np.fromiter((ids_of.setdefault(s, len(ids_of)) for s in strs), dtype=np.int32, count=len(strs))
    for s in ids_of:
        if "(" in s or "," in s or ")" in s:
            raise NotImplementedError("OddSth: the label %r contains '(', ',' or ')', so the reference's subtree "
                                      "strings are ambiguous for it" % s)
    try:
        rank = _value_ranks(labels)  # one order for all graphs: only the order within a graph matters
    except TypeError:
        rank = []
        gp = np.asarray(graph_ptr, dtype=np.int64)
        for g in range(len(gp) - 1):
            rank.extend(_value_ranks(labels[gp[g]:gp[g + 1]]))
    return ids, np.asarray(rank, dtype=np.int32), list(ids_of)


class OddSth(Kernel):
    """ODD-ST_h kernel (odd_sth.py; Da San Martino et al. 2012).  Every vertex v of a graph roots a DAG: the BFS from
    v over the out-neighbours, cut at depth h, ordered by Kahn's algorithm that pops the least (label value,
    insertion sequence).  A DAG node's identity is str(label) + "(" + its children's identities in ascending
    ordering + ")"; phi[f, g] counts the (root, node) pairs of graph g with identity f, and
    K[i, j] = sum_f C[f] phi[f, i] phi[f, j] with C[f] = phi[f, g0] for the first graph g0 that has f (the reference's
    `big_dag_append(..., merge_features=False)` keeps that graph's frequency).  The DAGs, the identities (hashed,
    verified and interned without building a string) and the exact integer Gram run on the device; K equals the
    reference's with ==.

    Vertices are the indices of an adjacency matrix or the symbols that occur in an edge of an edge dictionary; a
    vertex's neighbours come in ascending column order or in the order the edges were first listed, as in the
    reference's edge dictionary, and that order is part of the result.  Edge labels are ignored.  Labels are compared
    by value for the order and by str for the identity (1 and 1.0 tie in the order but are different features).  As
    in the reference, `transform` with normalize=True after `fit` (not `fit_transform`) raises AttributeError, and
    `diagonal()` is only defined after `transform`.  Deviations: a label whose str contains '(', ',' or ')', a graph
    of more than 4096 vertices, 2^30 or more (root, vertex) or (root, edge) pairs and a datasets.read_tu block (its
    edge sets carry no neighbour order) raise NotImplementedError; labels of one graph that cannot be compared raise
    TypeError."""

    _graph_format = "dictionary"

    def __init__(self, n_jobs=None, normalize=False, verbose=False, h=None):
        super().__init__(n_jobs=n_jobs, normalize=normalize, verbose=verbose)
        self.h = h
        self._initialized.update({"h": False})

    def initialize(self):
        """odd_sth.py:60-72."""
        if not self._initialized["n_jobs"]:
            if self.n_jobs is not None:
                warnings.warn("no implemented parallelization for OddSth")
            self._initialized["n_jobs"] = True
        if not self._initialized["h"]:
            if self.h is not None and (type(self.h) is not int or self.h <= 0):
                raise ValueError("h must be an integer bigger than zero")
            self.h_ = -1 if self.h is None else self.h
            self._initialized["h"] = True

    def parse_input(self, X):
        """odd_sth.py:74-127: the element checks, then the graphs packed with the edge dictionary's neighbour order."""
        if isinstance(X, Block) and X.mode == "core":  # a CoreFramework level: neighbours in the edge dictionary's order
            return self._fitted(X)
        if isinstance(X, Block):
            raise NotImplementedError("OddSth: a datasets.read_tu block does not carry the neighbour order of the "
                                      "reference's edge sets, which the result depends on; pass the list of graphs")
        if not isinstance(X, Iterable):
            raise TypeError("input must be an iterable\n")
        els = []
        for idx, x in enumerate(iter(X)):
            if isinstance(x, Graph):
                x = x.as_element()
            is_iter = isinstance(x, Iterable)
            if is_iter:
                x = list(x)
            if is_iter and len(x) == 0:
                warnings.warn("Ignoring empty element on index: " + str(idx))
                continue
            if not (is_iter and len(x) >= 2):
                raise TypeError(_ODD_ELEMENT_MSG)
            if type(x[0]) is dict and x[0] and all(type(d) is list for d in x[0].values()) and not all(x[0].values()):
                # {u: []}: u is a vertex without an edge-dictionary entry (graph.py:849-855)
                raise ValueError("vertex not inside edge dictionary")
            els.append([x[0], x[1]])
        if not els:
            raise ValueError("parsed input is empty")
        return self._fitted(pack(els, "sp", need_labels=True, len_ok=lambda n: n == 2, type_error_msg=_ODD_ELEMENT_MSG,
                                 keep_edge_order=True))

    @staticmethod
    def _fitted(block):
        ids, rank, strings = odd_label_tables(block.labels, block.graph_ptr)
        out = Fitted(block, ids, strings)
        out.rank = rank
        return out

    def fit_transform(self, X, y=None):
        self._method_calling = 2
        self.fit(X)
        K, xd, _ = self._odd_run(self.X.block, self.X.ids, self.X.rank, self.X.block.n_graphs)
        self._X_diag = xd
        return K

    def transform(self, X):
        """odd_sth.py:176-225: the fitted and the new graphs' identities in one dictionary, C from the first graph
        that has each identity (a fitted one for every identity that reaches K)."""
        self._method_calling = 3
        check_is_fitted(self, ["X"])
        if X is None:
            raise ValueError("transform input cannot be None")
        Y = self.parse_input(X)
        if self.normalize and getattr(self, "_X_diag", None) is None:
            # diagonal() of the reference reads self._phi_X, which it never sets
            raise AttributeError("'OddSth' object has no attribute '_phi_X'")
        # one label id per distinct str over both sides; ranks only order labels within a graph
        at = {s: i for i, s in enumerate(self.X.dictionary)}
        y_ids = np.array([at.setdefault(s, len(at)) for s in Y.dictionary], dtype=np.int32)[Y.ids]
        K, _, yd = self._odd_run(Block.concat(self.X.block, Y.block), np.concatenate([self.X.ids, y_ids]),
                                 np.concatenate([self.X.rank, Y.rank]), self.X.block.n_graphs)
        self._Y_diag = yd.reshape(-1, 1)
        self._is_transformed = True
        return K

    def diagonal(self):
        """odd_sth.py:227-255: (X diagonal, Y diagonal as a column) after `transform`."""
        check_is_fitted(self, ["_Y_diag"])
        if getattr(self, "_X_diag", None) is None:
            raise AttributeError("'OddSth' object has no attribute '_phi_X'")
        return self._X_diag, self._Y_diag

    def _odd_run(self, block, ids, rank, n_fit, want_matrix=True, device_ptr=None, row_range=None):
        """pack -> gk_odd_features (DAGs, identities, bit-plane tables) -> gk_gram (gram_path 14)."""
        with _run_engine(self) as eng:
            eng.pack(block.graph_ptr, block.row_ptr, block.col_idx, ids, None, None)
            self.stats_ = eng.odd_features(self.h_, rank)
            K, xd, yd = _gram_or_fold(self, eng, block.n_graphs, n_fit, want_matrix,
                                      normalize=bool(self.normalize) and want_matrix, device_ptr=device_ptr,
                                      row_range=row_range, stats=self.stats_)
            if getattr(self, "_keep_signatures", False):  # tests: the identities' signatures
                self.signatures_ = eng.odd_signatures()
        if self.verbose:
            print(type(self).__name__, self.stats_.as_dict())
        return K, xd, yd


# ------------------------------------------------------------------------------
# The eigen-decomposition of MultiscaleLaplacian's sampled blocks, by module-level name (the reference's numpy call):
# tests hand recorded eigenpairs back through it where a truncation boundary is nearly tied.
ml_eig = np.linalg.eig
_ML_POSITIVE = float("+1e-6")
_ML_NMAX = 128
_ML_ELEMENT_MSG = ("each element of X must be either a graph or an iterable with at least 1 and at most 3 elements\n")


def ml_truncate(K, P):
    """(v, w) of the reference's eig of the sample block K, its `argpartition(v, -P)[-P:]` cut and the 1e-6 filter:
    (eigenvalues kept, their eigenvectors as rows)."""
    v, w = ml_eig(K)
    v, w = np.real(v), np.real(w.T)
    vpos = np.argpartition(v, -P)[-P:]
    vpos = vpos[np.where(v[vpos] > _ML_POSITIVE)]
    return v[vpos], w[vpos]


class MultiscaleLaplacian(Kernel):
    """Multiscale Laplacian graph kernel (multiscale_laplacian.py; Kondor & Pan 2016), the fast FLG variant of the
    reference.  Per level l = 1 .. L every vertex's neighbourhood of radius l gives S = U^T (L_nb + heta I)^-1 U +
    gamma I over the previous level's features U, and the features of the next level are the FLG kernel values of the
    vertex against n_samples sampled vertices, projected on the top-P eigenvectors of the sampled block.  K is the FLG
    kernel of every graph's final S over its whole Laplacian.

    The samples are the reference's: the same list of (graph, vertex) pairs shuffled by `random_state_`, so a second
    `fit` draws new ones as the reference does.  The eigen-decompositions of the sampled blocks run on the host through
    `ml_eig` (numpy's eig, with the reference's argpartition and 1e-6 cut); every neighbourhood, record, projection and
    the Gram run on the device in fp64.  The device factors each matrix by Cholesky where the reference calls inv and
    eigvals, so K agrees with the reference to about 1e-11 relative rather than bit for bit; K is exactly symmetric and
    its diagonal is what `diagonal()` returns.

    Deviations (NotImplementedError): a non-symmetric adjacency matrix, a negative edge weight, gamma == 0 or heta == 0
    (the reference warns that it may crash; the warning is kept), a graph of more than 128 vertices, a feature width
    P' (eigenvalues kept) of 0 or above 32, more than 1024 samples.  A non-positive pivot met on the device raises an
    error rather than returning NaN."""

    _graph_format = "adjacency"

    def __init__(self, n_jobs=None, normalize=False, verbose=False, random_state=None, L=3, P=10, gamma=0.01,
                 heta=0.01, n_samples=50):
        super().__init__(n_jobs=n_jobs, normalize=normalize, verbose=verbose)
        self.random_state = random_state
        self.gamma = gamma
        self.heta = heta
        self.L = L
        self.P = P
        self.n_samples = n_samples
        self._initialized.update({"random_state": False, "gamma": False, "heta": False, "L": False,
                                  "n_samples": False, "P": False})

    def initialize(self):
        """multiscale_laplacian.py:86-131, in its order and with its errors."""
        super().initialize()
        if not self._initialized["random_state"]:
            self.random_state_ = check_random_state(self.random_state)
            self._initialized["random_state"] = True
        for name in ("gamma", "heta"):
            if not self._initialized[name]:
                val = getattr(self, name)
                if not isinstance(val, Real):
                    raise TypeError(name + " must be a real number")
                elif val == .0:
                    warnings.warn("with zero " + name + " the calculation may crash")
                elif val < 0:
                    raise TypeError(name + " must be positive")
                self._initialized[name] = True
        if not self._initialized["L"]:
            if type(self.L) is not int:
                raise TypeError("L must be an integer")
            elif self.L < 0:
                raise TypeError("L must be positive")
            self._initialized["L"] = True
        if not self._initialized["n_samples"]:
            if type(self.n_samples) is not int or self.n_samples <= 0:
                raise TypeError("n_samples must be a positive integer")
            self._initialized["n_samples"] = True
        if not self._initialized["P"]:
            if type(self.P) is not int or self.P <= 0:
                raise TypeError("P must be a positive integer")
            self._initialized["P"] = True

    # ---- input
    @staticmethod
    def _features(A, labels):
        try:
            phi = np.array([list(labels[i]) for i in range(A.shape[0])])
        except TypeError:
            raise TypeError("Features must be iterable and castable in total to a numpy array.")
        return A, phi

    def _elements(self, X):
        """(adjacency matrix, attribute matrix) of every element (multiscale_laplacian.py:154-186)."""
        from .packing import adjacency_and_labels
        if isinstance(X, Block):  # datasets.read_tu: the vertices that occur in an edge, with their attribute rows
            out = []
            gp = X.graph_ptr
            for g, (A, _) in enumerate(_block_adjacency(X, False)):
                rows = None if X.attrs is None else X.attrs[int(gp[g]):int(gp[g + 1])]
                out.append(self._features(A, rows if rows is not None else [0] * A.shape[0]))
            if not out:
                raise ValueError("parsed input is empty")
            return out
        if not isinstance(X, Iterable):
            raise TypeError("input must be an iterable\n")
        out = []
        for idx, x in enumerate(iter(X)):
            if isinstance(x, Graph):
                x = x.as_element()
            is_iter = isinstance(x, Iterable)
            if is_iter:
                x = list(x)
            if not (is_iter and len(x) in (0, 2, 3)):
                raise TypeError(_ML_ELEMENT_MSG)
            if len(x) == 0:
                warnings.warn("Ignoring empty element on index: " + str(idx))
                continue
            A, labels = adjacency_and_labels(x[0], x[1])
            out.append(self._features(A, labels))
        if not out:
            raise ValueError("parsed input is empty")
        return out

    def _check_scope(self, els):
        if self.gamma == 0 or self.heta == 0:
            raise NotImplementedError("MultiscaleLaplacian: gamma == 0 or heta == 0 has no Cholesky route")
        for A, _ in els:
            if A.shape[0] > _ML_NMAX:
                raise NotImplementedError("MultiscaleLaplacian: a graph of more than 128 vertices")
            if np.any(A < 0):
                raise NotImplementedError("MultiscaleLaplacian: a negative edge weight")
            if not np.array_equal(A, A.T):
                raise NotImplementedError("MultiscaleLaplacian: a non-symmetric adjacency matrix")

    def _ml_pipeline(self, eng, els, fit_rec=None):
        """multiscale_laplacian.py:188-310 on the device `eng`: fit (`_method_calling` 1) samples and keeps every
        level's basis, transform (3) applies them.  Leaves the Gram's records on `eng` (the fitted ones `fit_rec`
        first) and returns the packed graphs' final records."""
        sizes = [A.shape[0] for A, _ in els]
        gp = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
        # CSR of every graph's non-zero entries (diagonal included: it marks level-1 self-loops) with their weights
        rows, cols, vals = [], [], []
        for g, (A, _) in enumerate(els):
            ii, jj = np.nonzero(A)
            rows.append(ii + gp[g]); cols.append(jj + gp[g]); vals.append(A[ii, jj])
        rows = np.concatenate(rows) if rows else np.zeros(0, np.int64)
        cols = np.concatenate(cols) if cols else np.zeros(0, np.int64)
        vals = np.concatenate(vals) if vals else np.zeros(0)
        rp = np.concatenate([[0], np.cumsum(np.bincount(rows, minlength=int(gp[-1])))])
        phi = np.concatenate([np.asarray(p, dtype=np.float64).reshape(len(p), -1) for _, p in els])
        stats = {"host_eig_ms": 0.0}
        import time
        eng.pack(gp, rp, cols, None, vals, None)
        stats["begin"] = eng.ml_begin(self.L, self.gamma, self.heta, phi).as_dict()
        fit = self._method_calling == 1
        if fit:
            V = [(k, j) for k in range(len(els)) for j in range(sizes[k])]
            ns = min(len(V), self.n_samples)
            self.random_state_.shuffle(V)
            vs = V[:ns]
            phi_k = np.array([els[k][1][j, :] for (k, j) in vs])
            t0 = time.perf_counter()
            v, w = ml_truncate(phi_k.dot(phi_k.T), self.P)
            stats["host_eig_ms"] += (time.perf_counter() - t0) * 1e3
            ksi = w.dot(phi_k).T / np.sqrt(v)
            self._data_level = {0: ksi}
            self.samples_ = [vs]
        else:
            ksi = self._data_level[0]
        stats["project"] = [eng.ml_project(self._width_check(ksi)).as_dict()]
        width = ksi.shape[1]
        stats["levels"] = []
        for l in range(1, self.L + 1):
            if fit:
                self.random_state_.shuffle(V)
                vs = V[:ns]
                ids = np.array([gp[k] + j for k, j in vs], dtype=np.int32)
                rec, kss, s = eng.ml_level(l, width, samples=ids)
                t0 = time.perf_counter()
                v, w = ml_truncate(kss, self.P)
                stats["host_eig_ms"] += (time.perf_counter() - t0) * 1e3
                Q = w.T / np.sqrt(v)
                self._data_level[l] = (rec, Q)
                self.samples_.append(vs)
            else:
                rec, Q = self._data_level[l]
                _, _, s = eng.ml_level(l, width, samp_rec=rec)
            stats["levels"].append(s.as_dict())
            stats["project"].append(eng.ml_project(self._width_check(Q)).as_dict())
            width = Q.shape[1]
        recs, s = eng.ml_finish(width, fit_rec=fit_rec)
        stats["finish"] = s.as_dict()
        self.ml_stats_ = stats
        return recs

    @staticmethod
    def _width_check(Q):
        if Q.shape[1] == 0:
            raise NotImplementedError("MultiscaleLaplacian: no eigenvalue of the sampled block above 1e-6")
        return Q

    # ---- estimator protocol
    def fit(self, X, y=None):
        self._method_calling = 1
        self._is_transformed = False
        self.initialize()
        if X is None:
            raise ValueError("`fit` input cannot be None")
        self.__dict__.pop("_X_diag", None)
        self._ml_fit(X, want_matrix=False)
        return self

    def _ml_fit(self, X, want_matrix):
        els = self._elements(X)
        self._check_scope(els)
        with _lib.engine(getattr(self, "device_", None)) as eng:
            self.X = self._ml_pipeline(eng, els)
            K, xd, _ = eng.gram(len(self.X), normalize=bool(self.normalize) and want_matrix,
                                out=None if want_matrix else False)
        self._X_diag = xd
        return K

    def fit_transform(self, X, y=None):
        self._method_calling = 1  # fit_transform sets 2, and fit resets it to 1: the sampling route
        self._is_transformed = False
        self.initialize()
        if X is None:
            raise ValueError("`fit` input cannot be None")
        K = self._ml_fit(X, want_matrix=True)
        if self.normalize:
            self._warn_unnormalizable(self._X_diag)
        return K

    def transform(self, X):
        self._method_calling = 3
        check_is_fitted(self, ["X"])
        if X is None:
            raise ValueError("`transform` input cannot be None")
        els = self._elements(X)
        self._check_scope(els)
        nx = len(self.X)
        with _lib.engine(getattr(self, "device_", None)) as eng:
            Y = self._ml_pipeline(eng, els, fit_rec=self.X)
            K, xd, yd = eng.gram(nx + len(Y), n_fit=nx, normalize=bool(self.normalize))
        self._X_diag, self._Y_diag = xd, yd
        self._is_transformed = True
        if self.normalize:
            self._warn_unnormalizable(xd, yd)
        return K

    def diagonal(self):
        check_is_fitted(self, ["X"])
        if getattr(self, "_is_transformed", False):
            return self._X_diag, self._Y_diag
        return self._X_diag


# ------------------------------------------------------------------------------
_SVMT_NMAX = 128


def svm_theta_inner(x, y):
    """SvmTheta's default metric, the reference's `_inner`: np.inner(x, y)[0, 0], the product of the first levels."""
    return np.inner(x, y)[0, 0]


def svmt_distribute(n, subsets_size_range, n_samples):
    """{subset size: samples} for a graph of n vertices, as the reference's schedule: every size k from the smallest to
    min(largest, n) gets floor(n_samples * C(n, k) / sum of the C(n, k)) samples; what is left over is handed out one
    sample at a time from the largest size downwards, wrapping round, so each size gets rem // m more and the last
    rem % m sizes one beyond that.  Sizes left without a sample are omitted.  A graph below the smallest size raises
    ZeroDivisionError, as the reference does."""
    lo, hi = subsets_size_range
    sizes = np.arange(lo, min(hi, n) + 1)
    m = len(sizes)
    if m == 0:
        raise ZeroDivisionError("integer modulo by zero")
    share = np.array([binom(n, int(k)) for k in sizes], dtype=float)
    share = share / np.sum(share)
    count = np.floor(share * n_samples).astype(int)
    rem = max(int(n_samples - np.sum(count)), 0)
    count += rem // m
    if rem % m:
        count[m - rem % m:] += 1
    return {int(k): int(c) for k, c in zip(sizes, count) if c > 0}


class SvmTheta(Kernel):
    """SVM-theta kernel (svm_theta.py; Johansson et al. 2014).  Per graph: the smallest eigenvalue m of the 0/1
    adjacency (upper triangle mirrored), a one-class SVM fit on the adjacency scaled by 1 / -m with a unit diagonal,
    then phi[level] = the mean over sampled vertex subsets of that size of the sum of their alphas.  K[i, j] =
    metric(phi_i, phi_j); the default metric is the product of the first levels.

    The eigenvalue, libsvm's one-class SMO (restated with its rounding, so the alphas and iteration counts are the
    reference's), the subset sums and means (in numpy's summation order) and the Gram run on the device in fp64.  The
    subsets are the reference's: `RandomState.choice(n, level, replace=False)` restated in the library's host code on
    `random_state_`'s MT19937 stream, which then continues as the reference's does (a second fit, or a transform, draws
    after the earlier ones).  Any metric other than the default goes through the host pairwise driver.

    With the default subsets_size_range (2, 8) the first level gets no samples once a graph has 12 vertices or more,
    so the default kernel is 0 for such graphs; this is the reference's behaviour and is kept.

    Deviations (NotImplementedError): a graph of more than 128 vertices.  libsvm need not converge on the non-symmetric
    matrix of a directed graph, where the reference never returns; the device stops after 10^7 iterations with an
    error.

    `svmt_stats_` holds the stage times of the last run (ms): `h2d_ms` (masks, schedule and indexes), `eigenvalue_ms`,
    `smo_ms`, `host_draw_ms` (overlapping the two before it), `phi_ms`, `d2h_ms`."""

    _graph_format = "adjacency"
    # Not a parameter: set on an instance to keep, in `details_`, the last run's per-graph smallest eigenvalues (m),
    # alphas, SMO iteration counts (iters) and drawn indexes (drawn), for tests and diagnostics.
    _keep_details = False

    def __init__(self, n_jobs=None, normalize=False, verbose=False, random_state=None, n_samples=50,
                 subsets_size_range=(2, 8), metric=svm_theta_inner):
        super().__init__(n_jobs=n_jobs, normalize=normalize, verbose=verbose)
        self.n_samples = n_samples
        self.subsets_size_range = subsets_size_range
        self.metric = metric
        self.random_state = random_state
        self._initialized.update({"n_samples": False, "subsets_size_range": False, "metric": False,
                                  "random_state": False})

    def initialize(self):
        """svm_theta.py:70-99, in its order and with its errors."""
        super().initialize()
        if not self._initialized["n_samples"]:
            if self.n_samples <= 0 or type(self.n_samples) is not int:
                raise TypeError("n_samples must an integer be bigger than zero")
            self._initialized["n_samples"] = True
        if not self._initialized["subsets_size_range"]:
            r = self.subsets_size_range
            if (type(r) is not tuple or len(r) != 2 or any(type(i) is not int for i in r) or r[0] > r[1]
                    or r[0] <= 0):
                raise TypeError("subsets_size_range subset size rangemust be a tuple of two integers in increasing "
                                "order, bigger than 1")
            self._initialized["subsets_size_range"] = True
        if not self._initialized["metric"]:
            if not callable(self.metric):
                raise TypeError("metric between argumentsmust be a function")
            self._initialized["metric"] = True
        if not self._initialized["random_state"]:
            self.random_state_ = check_random_state(self.random_state)
            self._initialized["random_state"] = True

    def _elements(self, X):
        """Adjacency matrices of every element (svm_theta.py:121-151)."""
        from .packing import adjacency_and_labels
        if isinstance(X, Block):
            return [A for A, _ in _block_adjacency(X, False)]
        if not isinstance(X, Iterable):
            raise TypeError("input must be an iterable\n")
        out = []
        for idx, x in enumerate(iter(X)):
            if isinstance(x, Graph):
                x = x.as_element()
            is_iter = isinstance(x, Iterable)
            if is_iter:
                x = list(x)
            if not (is_iter and len(x) in (0, 1, 2, 3)):
                raise TypeError(_RW_ELEMENT_MSG)
            if len(x) == 0:
                warnings.warn("Ignoring empty element on index: " + str(idx))
                continue
            out.append(adjacency_and_labels(x[0])[0])
        if not out:
            raise ValueError("parsed input is empty")
        return out

    def _schedule(self, sizes):
        """Samples per (graph, level); a graph below the smallest level raises ZeroDivisionError after the draws of the
        graphs before it, as in the reference."""
        lo, hi = self.subsets_size_range
        counts = np.zeros((len(sizes), hi - lo + 1), dtype=np.int32)
        memo = {}
        for g, n in enumerate(sizes):
            if n not in memo:
                try:
                    memo[n] = svmt_distribute(n, self.subsets_size_range, self.n_samples)
                except ZeroDivisionError:
                    _lib.svmt_draw(self.random_state_, sizes[:g], lo, counts[:g])
                    raise
            for level, v in memo[n].items():
                counts[g, level - lo] = v
        return counts

    def _svmt_run(self, eng, X, fit_phi0=None):
        """phi of every graph of X on the device `eng`, drawing from random_state_; leaves the first levels after
        `fit_phi0` on `eng` for its Gram.  Returns the list of (L, 1) phi arrays."""
        els = self._elements(X)
        sizes = np.array([A.shape[0] for A in els], dtype=np.int32)
        if np.any(sizes > _SVMT_NMAX):
            raise NotImplementedError("SvmTheta: a graph of more than 128 vertices")
        counts = self._schedule(sizes)
        adj = np.zeros((int(sizes.sum()), 128), dtype=bool)
        o = 0
        for A in els:
            n = A.shape[0]
            M = A > 1e-10
            np.fill_diagonal(M, False)
            adj[o:o + n, :n] = M
            o += n
        masks = np.packbits(adj, axis=1, bitorder="little").view("<u4")
        eng.svmt_solve(sizes, masks)
        t0 = time.perf_counter()
        idx = _lib.svmt_draw(self.random_state_, sizes, self.subsets_size_range[0], counts)
        draw_ms = (time.perf_counter() - t0) * 1e3
        phi, det, s = eng.svmt_phi(self.subsets_size_range[0], counts, idx, fit_phi0=fit_phi0,
                                   details=self._keep_details)
        self.svmt_stats_ = {"n_graphs": len(sizes), "n_vertices": int(sizes.sum()), "h2d_ms": s.ms_h2d,
                            "eigenvalue_ms": s.ms_features, "smo_ms": s.ms_rw, "host_draw_ms": draw_ms,
                            "phi_ms": s.ms_combine, "d2h_ms": s.ms_d2h}
        if det is not None:
            self.details_ = dict(m=det[0], alpha=det[1], iters=det[2], drawn=idx, sizes=sizes)
        return [row.reshape(-1, 1) for row in phi]

    def parse_input(self, X):
        with _lib.engine(getattr(self, "device_", None)) as eng:
            return self._svmt_run(eng, X)

    def pairwise_operation(self, x, y):
        return self.metric(x, y)

    def _device_gram(self):
        return self.metric is svm_theta_inner

    def fit_transform(self, X, y=None):
        if not self._device_gram():
            return self._pairwise_fit_transform(X)
        self._method_calling = 2
        self._is_transformed = False
        self.initialize()
        if X is None:
            raise ValueError("`fit` input cannot be None")
        with _lib.engine(getattr(self, "device_", None)) as eng:
            self.X = self._svmt_run(eng, X)
            K, xd, _ = eng.gram(len(self.X), normalize=bool(self.normalize))
        self._X_diag = xd
        if self.normalize:
            self._warn_unnormalizable(xd)
        return K

    def transform(self, X):
        if not self._device_gram():
            return self._pairwise_transform(X)
        self._method_calling = 3
        check_is_fitted(self, ["X"])
        if X is None:
            raise ValueError("`transform` input cannot be None")
        nx = len(self.X)
        with _lib.engine(getattr(self, "device_", None)) as eng:
            Y = self._svmt_run(eng, X, fit_phi0=np.array([x[0, 0] for x in self.X]))
            K, xd, yd = eng.gram(nx + len(Y), n_fit=nx, normalize=bool(self.normalize))
        self._Y = Y
        self._X_diag, self._Y_diag = xd, yd
        self._is_transformed = True
        if self.normalize:
            self._warn_unnormalizable(xd, yd)
        return K

    def diagonal(self):
        return self._pairwise_diagonal()


_GS_KMAX = 6
# graphlet_sampling.py:185-187: isomorphism classes of graphs of k vertices, used when `a` is -1
_GS_CLASSES = {1: 1, 2: 2, 3: 4, 4: 8, 5: 19, 6: 53, 7: 209, 8: 1253, 9: 13599}


class GraphletSampling(Kernel):
    """Graphlet sampling kernel (graphlet_sampling.py; Shervashidze et al. 2009), the sampled route (`sampling` a
    dict).  Every graph gets n_samples draws on `random_state_`'s legacy MT19937 stream, as the reference makes them:
    a size r = randint(min(3, n), min(k, n) + 1) (no draw when that range is one size) and choice(n, r,
    replace=False); the draws are host code and the stream continues as the reference's does (a second fit, or a
    transform, draws after the earlier ones).  Each sample is the undirected graph induced on its vertices by A > 0 (a
    pair is an edge when either direction is, a diagonal entry a self-loop); its class up to isomorphism, the
    (graph, class) counts and the exact integer Gram run on the device.  A graph's count of a class is its number of
    samples of that class, plus one unless it is the first graph in input order with the class (the reference's
    bins); in a transform every class the fitted graphs have gets the plus one, and a class only the new graphs have
    is counted from its first new graph.  Those classes add nothing to K but enter the diagonal, so normalize divides
    by them too.  K equals the reference's with ==.

    Deviations (NotImplementedError): sampling=None (every connected k-vertex subset, the reference's ConSubg) has no
    device path; k > 6; a graph whose adjacency is not symmetric (the reference's `isomorphic` compares the directed
    edges after bliss's canonical labeling of the undirected graph, so its classes of directed samples depend on
    which labeling bliss picks).

    `gs_stats_` holds the stage times of the last run (ms): `host_draw_ms`, `class_table_ms`, `h2d_ms`,
    `classify_ms`, `columns_ms`, `gram_ms`."""

    _graph_format = "adjacency"

    def __init__(self, n_jobs=None, normalize=False, verbose=False, random_state=None, k=5, sampling=None):
        super().__init__(n_jobs=n_jobs, normalize=normalize, verbose=verbose)
        self.random_state = random_state
        self.k = k
        self.sampling = sampling
        self._initialized.update({"random_state": False, "k": False, "sampling": False})

    def initialize(self):
        """graphlet_sampling.py:121-223, in its order and with its errors and warnings."""
        if not self._initialized["n_jobs"]:
            if self.n_jobs is not None:
                warnings.warn("no implemented parallelization for GraphletSampling")
            self._initialized["n_jobs"] = True
        if not self._initialized["random_state"]:
            self.random_state_ = check_random_state(self.random_state)
            self._initialized["random_state"] = True
        if not self._initialized["k"]:
            if type(self.k) is not int:
                raise TypeError("k must be an int")
            if self.k > 10:
                warnings.warn("graphlets are too big - computation may be slow")
            elif self.k < 3:
                raise TypeError("k must be bigger than 3")
            self._initialized["k"] = True
        if not self._initialized["sampling"]:
            sampling, k = self.sampling, self.k
            if sampling is None:
                n_samples = None
            elif type(sampling) is dict:
                if "n_samples" in sampling:
                    n_samples = sampling["n_samples"]
                    args = [arg for arg in ["delta", "epsilon", "a"] if arg in sampling]
                    if len(args):
                        # the reference passes the names as the warning category, so this raises TypeError
                        warnings.warn("Number of samples defined as input, ignoring arguments:", ", ".join(args))
                elif "delta" in sampling or "epsilon" in sampling or "a" in sampling:
                    delta = sampling.get("delta", 0.05)
                    epsilon = sampling.get("epsilon", 0.05)
                    a = sampling.get("a", -1)
                    if delta > 1 or delta < 0:
                        raise TypeError("delta must be in the range (0,1)")
                    if epsilon > 1 or epsilon < 0:
                        raise TypeError("epsilon must be in the range (0,1)")
                    if type(a) is not int:
                        raise TypeError("a must be an integer")
                    elif a == 0:
                        raise TypeError("a cannot be zero")
                    elif a < -1:
                        raise TypeError("negative a smaller than -1 have no meaning")
                    if a == -1:
                        if k > 9:
                            warnings.warn("warning for such size number of isomorphisms is not known - "
                                          "interpolation on know values will be used")
                            from scipy.interpolate import interp1d
                            a = interp1d(list(_GS_CLASSES.keys()), list(_GS_CLASSES.values()), kind="cubic")(k)
                        else:
                            a = _GS_CLASSES[k]
                    n_samples = math.ceil(2 * (a * np.log10(2) + np.log10(1 / delta)) / (epsilon ** 2))
                else:
                    raise ValueError("sampling doesn't have a valid dictionary format")
            else:
                raise TypeError("sampling can either be a dictionary or None")
            self.k_ = k
            self.n_samples_ = n_samples
            self._initialized["sampling"] = True

    def _check_scope(self):
        if self.n_samples_ is None:
            raise NotImplementedError("GraphletSampling: sampling=None (every connected k-vertex subset) has no device "
                                      "path; pass a sampling dictionary")
        if self.k_ > _GS_KMAX:
            raise NotImplementedError("GraphletSampling: graphlets of more than 6 vertices (k = %d)" % self.k_)
        n = self.n_samples_
        if type(n) is not int and not isinstance(n, np.integer):
            raise TypeError("'%s' object cannot be interpreted as an integer" % type(n).__name__)
        return max(int(n), 0)

    def _elements(self, X):
        """0/1 adjacency (A > 0) of every element, rows in sorted vertex order (graphlet_sampling.py:378-398)."""
        from .packing import adjacency_and_labels
        if isinstance(X, Block):
            return [A > 0 for A, _ in _block_adjacency(X, False)]
        if not isinstance(X, Iterable):
            raise TypeError("input must be an iterable\n")
        out = []
        for idx, x in enumerate(iter(X)):
            if isinstance(x, Graph):
                x = x.as_element()
            is_iter = isinstance(x, Iterable)
            if is_iter:
                x = list(x)
            if not (is_iter and len(x) in (0, 1, 2, 3)):
                raise TypeError("each element of X must be either a graph or an iterable with at least 1 and at most "
                                "3 elements\n")
            if len(x) == 0:
                warnings.warn("Ignoring empty element on index: " + str(idx))
                continue
            out.append(adjacency_and_labels(x[0])[0] > 0)
        if not out:
            raise ValueError("parsed input is empty")
        return out

    @staticmethod
    def _csr(mats):
        sizes = np.array([A.shape[0] for A in mats], dtype=np.int64)
        gp = np.zeros(len(mats) + 1, dtype=np.int64)
        gp[1:] = np.cumsum(sizes)
        rows, cols = [], []
        for A, o in zip(mats, gp[:-1]):
            r, c = np.nonzero(A)
            rows.append(r + o)
            cols.append(c + o)
        r = np.concatenate(rows) if rows else np.zeros(0, dtype=np.int64)
        c = np.concatenate(cols) if cols else np.zeros(0, dtype=np.int64)
        rp = np.zeros(gp[-1] + 1, dtype=np.int64)
        np.add.at(rp, r + 1, 1)
        return sizes, gp, np.cumsum(rp), c

    def _gs_run(self, new, fit_csr=None, fit_counts=None, want_matrix=True, device_ptr=None, row_range=None):
        """Draw for the graphs `new`, classify and count them after the fitted graphs (fit_csr, their counts), and
        return (K, xdiag, ydiag, counts of every graph)."""
        n_samples = self._check_scope()
        if any(not np.array_equal(A, A.T) for A in new):
            raise NotImplementedError("GraphletSampling: a graph with a non-symmetric adjacency matrix (the reference's "
                                      "classes of directed samples depend on bliss's canonical labeling)")
        sizes, gp, rp, ci = self._csr(new)
        t0 = time.perf_counter()
        samp_size, idx = _lib.gs_draw(self.random_state_, sizes, self.k_, n_samples)
        draw_ms = (time.perf_counter() - t0) * 1e3
        samp_off = np.arange(len(new) + 1, dtype=np.int64) * n_samples
        if fit_csr is not None:
            fs, fgp, frp, fci = fit_csr
            nx = len(fs)
            gp = np.concatenate([fgp, fgp[-1] + gp[1:]])
            rp = np.concatenate([frp, frp[-1] + rp[1:]])
            ci = np.concatenate([fci, fgp[-1] + ci])
        else:
            nx = len(new)
        N = len(gp) - 1
        with _lib.engine(getattr(self, "device_", None)) as eng:
            eng.pack(gp, rp, ci)
            st = eng.gs_features(self.k_, nx, N - len(new), samp_off, samp_size, idx,
                                 prior=None if fit_counts is None else fit_counts[:, :3])
            counts = eng.gs_counts()
            gst = _lib.GkStats()
            K, xd, yd = eng.gram(N, n_fit=nx, normalize=bool(self.normalize) and want_matrix,
                                 out=None if want_matrix else False, device_ptr=device_ptr, row_range=row_range,
                                 stats=gst)
        self.stats_ = st
        self.gs_stats_ = {"n_graphs": N, "n_samples": int(len(samp_size)), "host_draw_ms": draw_ms,
                          "class_table_ms": st.ms_hash, "h2d_ms": st.ms_h2d, "classify_ms": st.ms_features,
                          "columns_ms": st.ms_columns, "gram_ms": gst.ms_total}
        if self.verbose:
            print(type(self).__name__, self.gs_stats_)
        return K, xd, yd, counts

    def fit(self, X, y=None):
        self._is_transformed = False
        self._method_calling = 1
        self.initialize()
        if X is None:
            raise ValueError("`fit` input cannot be None")
        self._fit(X, want_matrix=False)
        return self

    def _fit(self, X, want_matrix):
        els = self._elements(X)
        K, xd, _, counts = self._gs_run(els, want_matrix=want_matrix)
        self._fit_csr = self._csr(els)
        self._nx = len(els)
        self.X = counts
        for a in ("_X_diag", "_Y_diag", "_phi_X"):
            self.__dict__.pop(a, None)
        return K, xd

    def fit_transform(self, X, y=None):
        self._method_calling = 2
        self._is_transformed = False
        self.initialize()
        if X is None:
            raise ValueError("`fit` input cannot be None")
        K, xd = self._fit(X, want_matrix=True)
        self._X_diag = xd
        self._phi_X = True
        return K

    def transform(self, X):
        self._method_calling = 3
        check_is_fitted(self, ["X"])
        if X is None:
            raise ValueError("transform input cannot be None")
        els = self._elements(X)
        K, xd, yd, counts = self._gs_run(els, fit_csr=self._fit_csr, fit_counts=self.X)
        self._ny = len(els)
        self.Y_ = counts[counts[:, 0] >= self._nx]
        self._X_diag, self._Y_diag = xd, yd
        self._phi_X = True
        self._is_transformed = True
        return K

    def diagonal(self):
        """graphlet_sampling.py:333-371: the X diagonal, and the Y diagonal after `transform`."""
        check_is_fitted(self, ["_phi_X"])
        if getattr(self, "_is_transformed", False):
            return self._X_diag, self._Y_diag
        return self._X_diag


_WL_GRAPH_BASES = (PyramidMatch, NeighborhoodSubgraphPairwiseDistance, OddSth, SubgraphMatching)
_HC_GRAPH_BASES = (PyramidMatch, NeighborhoodSubgraphPairwiseDistance, SubgraphMatching)
