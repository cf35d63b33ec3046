"""CoreFramework (grakel/kernels/core_framework.py:23-400) on the device engine.

The reference computes, for every core level i = max_core .. min_core+1, the base kernel on the
i-core subgraphs of the graphs that have one, and scatter-adds the per-level matrices
(core_framework.py:177-223).  Here all subgraphs of all levels are packed as separate graphs of ONE
block; vertex labels are tagged with their core level, so that no feature column is shared between
levels (each reference level has its own base-kernel instance, i.e. its own dictionaries); the C-ABI
row map (gk_set_row_map) sends every subgraph back to its graph's row, and one Gram over the joint
feature block equals the reference's sum over levels.  Base kernels: ShortestPath (the reference
default), WeisfeilerLehman (over VertexHistogram / ShortestPath), VertexHistogram.

NeighborhoodHash, OddSth, WeisfeilerLehmanOptimalAssignment and SubgraphMatching (ke=None) have Grams that are not a
sum of products of per-feature counts, so their levels cannot share one block.  They take the reference's own
structure: for every core level, from the largest down, a fresh base kernel is fitted on the level's subgraphs (built
in the reference's get_subgraph shape), its un-normalised K is computed on the device and scattered into the rows and
columns of the graphs that have such a subgraph (gk_core_level_add), and only the final sum crosses to the host.
"""
from __future__ import annotations

import time
import warnings
from collections.abc import Iterable

import numpy as np
from sklearn.utils.validation import check_is_fitted

from . import _lib
from .kernels import (CoreLevel, Kernel, NeighborhoodHash, OddSth, ShortestPath, SubgraphMatching, VertexHistogram,
                      WeisfeilerLehman, WeisfeilerLehmanOptimalAssignment, parse_base_kernel)
from .packing import Block, Graph, adjacency_and_order, label_ids, pack


def core_numbers(block):
    """Core number of every vertex of a packed block (Batagelj-Zaversnik result of
    core_framework.py:378-409, computed by vectorised peeling).  A self loop counts as one neighbour
    that is never removed before its vertex, as in the reference's neighbour lists."""
    V = block.n_vertices
    rp = block.row_ptr.astype(np.int64)
    ci = block.col_idx.astype(np.int64)
    deg = np.diff(rp)
    src = np.repeat(np.arange(V, dtype=np.int64), deg)
    cur = deg.copy()
    core = np.zeros(V, dtype=np.int64)
    alive = np.ones(V, dtype=bool)
    k, remaining = 0, V
    while remaining:
        rem = alive & (cur <= k)
        n_rem = int(rem.sum())
        if n_rem == 0:
            k = max(k + 1, int(cur[alive].min()))
            continue
        core[rem] = k
        alive[rem] = False
        remaining -= n_rem
        m = rem[src] & alive[ci]
        if m.any():
            np.subtract.at(cur, ci[m], 1)
    return core


def core_subgraph_block(block, core, tag_labels=True):
    """All non-empty i-core subgraphs (i = max core .. 0) of a block as one block.

    Returns (virtual block, row index of every virtual graph, max core number).  Labels become
    (level, label) pairs; weights and attributes are carried over."""
    N, V = block.n_graphs, block.n_vertices
    gp = block.graph_ptr.astype(np.int64)
    rp = block.row_ptr.astype(np.int64)
    ci = block.col_idx.astype(np.int64)
    deg = np.diff(rp)
    src = np.repeat(np.arange(V, dtype=np.int64), deg)
    vgraph = np.repeat(np.arange(N, dtype=np.int64), np.diff(gp))
    max_core = int(core.max()) if V else 0
    g_ptr, r_ptr, cols, w_parts, labels, rows = [np.zeros(1, dtype=np.int64)], [np.zeros(1, dtype=np.int64)], [], [], [], []
    v_off = e_off = 0
    for level in range(max_core, -1, -1):
        keep = core >= level
        newid = np.cumsum(keep) - 1
        em = keep[src] & keep[ci]
        nv = int(keep.sum())
        sizes = np.bincount(vgraph[keep], minlength=N)
        present = sizes > 0
        g_ptr.append(v_off + np.cumsum(sizes[present]))
        rows.append(np.nonzero(present)[0])
        r_ptr.append(e_off + np.cumsum(np.bincount(newid[src[em]], minlength=nv)))
        cols.append(newid[ci[em]] + v_off)
        if block.weights is not None:
            w_parts.append(block.weights[em])
        if block.labels is not None:
            kept = np.nonzero(keep)[0]
            labels.extend(((level, block.labels[v]) if tag_labels else block.labels[v]) for v in kept.tolist())
        v_off += nv
        e_off += int(em.sum())
    vb = Block(np.concatenate(g_ptr), np.concatenate(r_ptr), np.concatenate(cols) if cols else np.zeros(0, dtype=np.int64),
               np.concatenate(w_parts) if block.weights is not None else None,
               labels if block.labels is not None else None, None, block.all_adjacency)
    return vb, np.concatenate(rows).astype(np.int32), max_core


_FOLD_BASES = (NeighborhoodHash, OddSth, WeisfeilerLehmanOptimalAssignment, SubgraphMatching)


def level_blocks(block, core):
    """The reference's per-level inputs (core_framework.py:177-199) as blocks compacted from the block packed once: for
    every core level i = max core .. 0, the indices of the graphs with a vertex of core >= i and one block (mode
    "core") of their i-core subgraphs.  It holds what Graph.get_subgraph keeps of the dictionary format of
    Graph(x, "adjacency"): every kept vertex in matrix order, its kept neighbours in ascending order (the edge
    dictionary's), the weights and the vertex labels; the edge labels go to index_edge_labels there, which a dictionary
    reader never sees (graph.py:1467-1477).  Returns [(level, indexes, block)]."""
    N, V = block.n_graphs, block.n_vertices
    gp = block.graph_ptr.astype(np.int64)
    rp = block.row_ptr.astype(np.int64)
    ci = block.col_idx.astype(np.int64)
    src = np.repeat(np.arange(V, dtype=np.int64), np.diff(rp))
    vgraph = np.repeat(np.arange(N, dtype=np.int64), np.diff(gp))
    labels = block.labels
    max_core = int(core.max()) if V else 0
    out = []
    for level in range(max_core, -1, -1):
        keep = core >= level
        kept = np.nonzero(keep)[0]
        newid = np.cumsum(keep) - 1
        em = keep[src] & keep[ci]
        sizes = np.bincount(vgraph[keep], minlength=N)
        present = np.nonzero(sizes)[0]
        if labels is None:
            lab = None
        elif isinstance(labels, np.ndarray):
            lab = labels[kept].tolist()
        else:
            lab = [labels[v] for v in kept.tolist()]
        lb = Block(np.concatenate([[0], np.cumsum(sizes[present])]),
                   np.concatenate([[0], np.cumsum(np.bincount(newid[src[em]], minlength=len(kept)))]),
                   newid[ci[em]], None if block.weights is None else block.weights[em], lab)
        lb.mode = "core"
        out.append((level, present, lb))
    return out


def _labelled_everywhere(X, block, core, max_core):
    """Whether every level subgraph of every graph keeps an edge that carries an edge label: the reference's
    SubgraphMatching reads a subgraph's edge labels even with ke=None and raises without one.  Labels are keyed by
    the matrix indices of Graph(x, "adjacency") (matrix order, or the sorted symbols that occur in an edge)."""
    gp = block.graph_ptr.astype(np.int64)
    pu, pv = [], []
    for g, x in enumerate(X):
        if isinstance(x, Graph):
            x = x.as_element()
        x = list(x)
        el = x[2] if len(x) >= 3 and x[2] else {}
        _, order = adjacency_and_order(x[0])
        at = {s: i for i, s in enumerate(order)}
        for (u, v) in el:
            if u in at and v in at:
                pu.append(gp[g] + at[u])
                pv.append(gp[g] + at[v])
    pu, pv = np.array(pu, dtype=np.int64), np.array(pv, dtype=np.int64)
    vgraph = np.repeat(np.arange(block.n_graphs), np.diff(gp))
    for level in range(max_core, -1, -1):
        present = np.unique(vgraph[core >= level])
        ok = np.minimum(core[pu], core[pv]) >= level if len(pu) else np.zeros(0, dtype=bool)
        if not np.isin(present, vgraph[pu[ok]]).all():
            return False
    return True


class _FoldedCores:
    def __init__(self, levels, n_rows, max_core):
        self.levels, self.n_rows, self.max_core = levels, n_rows, max_core


class _FittedCores:
    def __init__(self, vblock, ids, rows, dictionary, n_rows, max_core):
        self.block, self.ids, self.rows, self.dictionary, self.n_rows, self.max_core = vblock, ids, rows, dictionary, n_rows, max_core


class CoreFramework(Kernel):
    """The core kernel framework (core_framework.py:23-400)."""

    _graph_format = "dictionary"
    _nan_to_num = True

    def __init__(self, n_jobs=None, verbose=False, normalize=False, min_core=-1, base_graph_kernel=None):
        super().__init__(n_jobs=n_jobs, verbose=verbose, normalize=normalize)
        # core_framework.py:50: the reference stores -1 whatever the argument says; results must match
        # the reference's, so the same is done here (sklearn clone/get_params then agree as well).
        self.min_core = -1
        self.base_graph_kernel = base_graph_kernel
        self._initialized.update({"min_core": False, "base_graph_kernel": False})

    def initialize(self):
        super().initialize()
        if not self._initialized["base_graph_kernel"]:  # core_framework.py:59-88
            base, params = parse_base_kernel(
                self, ShortestPath, (ShortestPath, WeisfeilerLehman, VertexHistogram) + _FOLD_BASES,
                "grakel_b200 runs CoreFramework over ShortestPath, WeisfeilerLehman, VertexHistogram, NeighborhoodHash, "
                "OddSth, WeisfeilerLehmanOptimalAssignment or SubgraphMatching; other base kernels are outside the "
                "device hot path", copy=True)
            if base is SubgraphMatching and params.get("ke", SubgraphMatching().ke) is not None:
                # a level subgraph keeps its edge labels under the original vertex ids while the adjacency view
                # renumbers the vertices, so the reference's edge kernel reads labels of other edges or fails
                raise NotImplementedError("CoreFramework over SubgraphMatching needs ke=None: the reference's level "
                                          "subgraphs do not carry usable edge labels")
            self.base_graph_kernel_ = base
            self.params_ = params
            self._base = base(**params)  # validates the parameters exactly like the reference's per-level instances
            self._base.initialize()
            self._fold = base in _FOLD_BASES
            self._initialized["base_graph_kernel"] = True
        if not self._initialized["min_core"]:
            if type(self.min_core) is not int or self.min_core < -1:
                raise TypeError("'min_core' must be an integer bigger than -1")
            self._initialized["min_core"] = True

    # ---- host side ------------------------------------------------------------
    def _pack(self, X):
        if not isinstance(X, Iterable):
            raise TypeError("input must be an iterable\n")
        base = self.base_graph_kernel_
        need_labels = not (base is ShortestPath and not self.params_.get("with_labels", True))
        # every element becomes Graph(x[0], x[1], x[2], "adjacency") first (core_framework.py:133-139):
        # the vertex set is the graph's own (matrix order / sorted symbols that occur in an edge)
        block = pack(X, "sp", need_labels=need_labels, len_ok=lambda n: n >= 1, want_weights=base is not VertexHistogram)
        if block.weights is not None and np.any(block.weights != np.rint(block.weights)):
            raise NotImplementedError("non-integer edge weights are supported with Floyd-Warshall semantics only")
        core = core_numbers(block)
        return core_subgraph_block(block, core) + (block.n_graphs,)

    def _fold_input(self, X):
        """The level blocks of X for a fold base (the reference's parse_input up to the base kernel calls)."""
        if not isinstance(X, Iterable):
            raise TypeError("input must be an iterable\n")
        t = time.perf_counter()
        X = list(X)
        need_labels = not (self.base_graph_kernel_ is SubgraphMatching and self._base.kv is None)
        block = pack(X, "sp", need_labels=need_labels, len_ok=lambda n: n >= 1, want_weights=True)
        core = core_numbers(block)
        max_core = int(core.max()) if block.n_vertices else 0
        if max_core <= self.min_core:
            raise ValueError("The maximum core equals the min_core boundary set in init.")
        if self.base_graph_kernel_ is SubgraphMatching and not _labelled_everywhere(X, block, core, max_core):
            raise ValueError("Graph does not have any labels for edges.")
        data = _FoldedCores(level_blocks(block, core), block.n_graphs, max_core)
        self.stage_times_ = {"levels": time.perf_counter() - t, "base": 0.0, "fold": 0.0}
        return data

    def _fold_levels(self, data, fit):
        """Run the base kernel of every level and fold its K into the device sum (fit: fit_transform, else transform).
        Returns (K un-normalised, its diagonal when fit)."""
        base = self.base_graph_kernel_
        n_cols = data.n_rows if fit else self._nx
        t = time.perf_counter()
        with _lib.engine(getattr(self, "device_", None)) as eng:
            eng.core_sum_begin(data.n_rows, n_cols, fit)
            for level, idx, lb in data.levels:
                if fit:
                    bk = self.X[level] = base(**self.params_)
                    cols = idx
                elif self._max_core_number < level or self._fit_indexes[level].shape[0] == 0:
                    if len(idx) > 0:  # the reference's dummy kernel: only its diagonal is read
                        bk = self._dummy_kernel[level] = base(**self.params_)
                        bk.fit(lb)
                    continue
                else:
                    bk, cols = self.X[level], self._fit_indexes[level]
                bk._core_level = CoreLevel(eng, level, idx, cols, self.stage_times_)
                try:
                    bk.fit_transform(lb) if fit else bk.transform(lb)
                finally:
                    del bk._core_level
            t_fetch = time.perf_counter()
            K, kd = eng.wl_level_sum_fetch(data.n_rows, n_cols, want_kdiag=fit)
        st = self.stage_times_
        st["fold"] += time.perf_counter() - t_fetch
        st["base"] = time.perf_counter() - t - st["fold"]
        return K, kd

    def _fold_fit(self, X, transform):
        self.X = {}
        data = self._fold_input(X)
        self._nx, self._max_core_number = data.n_rows, data.max_core
        self._fit_indexes = {level: idx for level, idx, _ in data.levels}
        self.__dict__.pop("_X_diag", None)
        if not transform:
            for level, idx, lb in data.levels:
                self.X[level] = self.base_graph_kernel_(**self.params_)
                self.X[level].fit(lb)
            return None
        K, kd = self._fold_levels(data, True)
        self._X_diag = kd
        if self.normalize:
            with np.errstate(divide="ignore", invalid="ignore"):
                K = np.nan_to_num(np.divide(K, np.sqrt(np.outer(kd, kd))))
        return K

    def _fold_transform(self, X):
        data = self._fold_input(X)
        self._dummy_kernel = {}
        self._t_nx, self._max_core_number_trans = data.n_rows, data.max_core
        self._transform_indexes = {level: idx for level, idx, _ in data.levels}
        K, _ = self._fold_levels(data, False)
        self._is_transformed = True
        if self.normalize:
            X_diag, Y_diag = self._fold_diagonal()
            with np.errstate(divide="ignore", invalid="ignore"):
                K /= np.sqrt(np.outer(Y_diag, X_diag))
            K = np.nan_to_num(K)
        return K

    def _fold_diagonal(self):
        """core_framework.py:313-375, level order and all."""
        Y_diag = None
        if hasattr(self, "_X_diag"):
            if self._is_transformed:
                Y_diag = np.zeros(shape=(self._t_nx,))
                for i in range(min(self._max_core_number_trans, self._max_core_number), self.min_core, -1):
                    tidx = self._transform_indexes[i]
                    if tidx.shape[0] > 0:
                        Y_diag[tidx] += self.X[i].diagonal()[1]
        else:
            X_diag = np.zeros(shape=(self._nx,))
            if self._is_transformed:
                max_core_number = min(self._max_core_number_trans, self._max_core_number)
                Y_diag = np.zeros(shape=(self._t_nx,))
                for i in range(max_core_number, self.min_core, -1):
                    fidx, tidx = self._fit_indexes[i], self._transform_indexes[i]
                    if tidx.shape[0] > 0 and fidx.shape[0] > 0:
                        x, y = self.X[i].diagonal()
                        X_diag[fidx] += x
                        Y_diag[tidx] += y
                if max_core_number < self._max_core_number:
                    for i in range(self._max_core_number, self._max_core_number_trans, -1):
                        fidx = self._fit_indexes[i]
                        if fidx.shape[0] > 0:
                            X_diag[fidx] += self.X[i].diagonal()
            else:
                for i in range(self._max_core_number, self.min_core, -1):
                    fidx = self._fit_indexes[i]
                    if fidx.shape[0] > 0:
                        X_diag[fidx] += self.X[i].diagonal()
            self._X_diag = X_diag
        if self._is_transformed:
            for idx, bk in self._dummy_kernel.items():
                Y_diag[self._transform_indexes[idx]] += bk.diagonal()
            return self._X_diag, Y_diag
        return self._X_diag

    def parse_input(self, X):
        vb, rows, max_core, n = self._pack(X)
        if max_core <= self.min_core:
            raise ValueError("The maximum core equals the min_core boundary set in init.")
        sort_new = self.base_graph_kernel_ is WeisfeilerLehman
        if vb.labels is None:
            ids, dictionary = None, {}
        elif self._method_calling in (1, 2):
            ids, dictionary = label_ids(vb.labels, None, sort_new=sort_new)
        else:
            ids, _ = label_ids(vb.labels, self.X.dictionary, sort_new=sort_new)
            dictionary = self.X.dictionary
        return _FittedCores(vb, ids, rows, dictionary, n, max_core)

    # ---- device side ----------------------------------------------------------
    def _device_features(self, eng):
        base, b = self.base_graph_kernel_, self._base
        if base is ShortestPath:
            return eng.sp_features(with_labels=bool(b.with_labels))
        if base is VertexHistogram:
            return eng.wl_features(0)
        if b._base_graph_kernel is ShortestPath:
            return eng.wl_sp_features(b._n_iter - 1)
        if b._base_graph_kernel is not VertexHistogram:
            raise NotImplementedError("CoreFramework over WeisfeilerLehman needs the subtree or ShortestPath base kernel")
        return eng.wl_features(b._n_iter - 1)

    def _run_cores(self, block, ids, rows, n_rows, n_fit, want_matrix=True):
        with _lib.engine(getattr(self, "device_", None)) as eng:
            eng.pack(block.graph_ptr, block.row_ptr, block.col_idx, ids, block.weights, block.attrs)
            eng.set_row_map(n_rows, rows)
            self.stats_ = self._device_features(eng)
            K, xd, yd = eng.gram(n_rows, n_fit=n_fit, normalize=bool(self.normalize) and want_matrix,
                                 nan_to_num=True, out=None if want_matrix else False, stats=self.stats_)
        return K, xd, yd

    def fit(self, X, y=None):
        self._is_transformed = False
        self._method_calling = 1
        self.initialize()
        if X is None:
            raise ValueError("`fit` input cannot be None")
        if getattr(self, "_fold", False):
            self._fold_fit(X, transform=False)
            return self
        self.X = self.parse_input(X)
        self._nx = self.X.n_rows
        self._max_core_number = self.X.max_core
        if hasattr(self, "_X_diag"):
            delattr(self, "_X_diag")
        return self

    def fit_transform(self, X, y=None):
        self._method_calling = 2
        self._is_transformed = False
        self.initialize()
        if X is None:
            raise ValueError("transform input cannot be None")
        if getattr(self, "_fold", False):
            return self._fold_fit(X, transform=True)
        self.X = self.parse_input(X)
        self._nx = self.X.n_rows
        self._max_core_number = self.X.max_core
        K, xd, _ = self._run_cores(self.X.block, self.X.ids, self.X.rows, self._nx, self._nx)
        self._X_diag = xd
        return K

    def transform(self, X):
        self._method_calling = 3
        check_is_fitted(self, ["X"])
        if X is None:
            raise ValueError("transform input cannot be None")
        if getattr(self, "_fold", False):
            return self._fold_transform(X)
        Y = self.parse_input(X)
        block = Block.concat(self.X.block, Y.block)
        ids = None if self.X.ids is None else np.concatenate([self.X.ids, Y.ids])
        rows = np.concatenate([self.X.rows, Y.rows + self._nx]).astype(np.int32)
        K, xd, yd = self._run_cores(block, ids, rows, self._nx + Y.n_rows, self._nx)
        self._X_diag, self._Y_diag = xd, yd
        self._is_transformed = True
        return K

    def diagonal(self):
        check_is_fitted(self, ["X"])
        if getattr(self, "_fold", False):
            return self._fold_diagonal()
        if not hasattr(self, "_X_diag"):
            _, self._X_diag, _ = self._run_cores(self.X.block, self.X.ids, self.X.rows, self._nx, self._nx,
                                                 want_matrix=False)
        if getattr(self, "_is_transformed", False):
            return self._X_diag, self._Y_diag
        return self._X_diag

