"""Host-side input normalisation: reference-style graph inputs -> one CSR block.

Mirrors the *behaviour* of grakel.Graph for the parts the hot path touches
(graph.py:147-230 build_graph, :912-1053 _import_adjacency/_import_dictionary,
:1542-1709 is_adjacency/is_edge_dictionary, :689-772 get_labels):

* adjacency input (2-D ndarray, scipy sparse, list of number lists): vertices are
  0..n-1, an edge is an entry > 0 (graph.py:963, 1198);
* edge-dictionary input in five spellings: {(u,v): w}, {u: [v, ...]},
  {u: {v: w}}, iterable of (u,v), iterable of (u,v,w); vertices are sorted
  symbols (graph.py:902-905); every listed edge is kept, whatever its weight;
* node labels: dict keyed by vertex symbol (dictionary input) or index
  (adjacency input).

The result is a `Block`: int32 CSR over all graphs (neighbour ids are global
vertex ids), one Python label object per vertex, optional fp64 edge weights.
"""
from __future__ import annotations

import numbers
import os
import warnings
from collections.abc import Iterable
from itertools import chain

import numpy as np

try:  # CPython-level packer for the commonest spelling (csrc/fastpack.c, built by csrc/build.sh); optional
    from . import _fastpack
except Exception:  # pragma: no cover
    _fastpack = None

try:  # scipy is a hard dependency of the reference; optional here
    from scipy.sparse import issparse
except Exception:  # pragma: no cover
    def issparse(x):
        return False


class Graph:
    """Minimal stand-in for grakel.Graph as an *input carrier*: kernels accept
    `Graph(initialization_object, node_labels, edge_labels)` instances wherever
    the reference does (kernel.py:377-378, weisfeiler_lehman.py:171-179)."""

    def __init__(self, initialization_object=None, node_labels=None, edge_labels=None, graph_format="auto",
                 construct_labels=False):
        if graph_format not in ("adjacency", "dictionary", "auto", "all"):
            raise ValueError('Invalid graph format.\nValid graph formats are "all", "dictionary", "adjacency", "auto"')
        if initialization_object is None and graph_format == "auto":
            raise ValueError("no initialization object - format must not be auto")
        if initialization_object is not None and classify(initialization_object) is None:
            raise ValueError("Unsupported input type. For more information check the documentation, concerning "
                             "valid input types for graph type object.")
        self.initialization_object = initialization_object
        self.node_labels = node_labels
        self.edge_labels = edge_labels
        self.graph_format = graph_format
        self.construct_labels = construct_labels

    def as_element(self):
        return [self.initialization_object, self.node_labels if self.node_labels is not None else {},
                self.edge_labels if self.edge_labels is not None else {}]


def classify(g):
    """'adjacency', a dictionary spelling name, or None (graph.py:1542-1709)."""
    if isinstance(g, np.ndarray) and g.ndim == 2:
        return "adjacency"
    if issparse(g):
        return "adjacency"
    if type(g) is list and all(isinstance(r, list) and all(isinstance(x, numbers.Number) for x in r) for r in g):
        return "adjacency"
    if type(g) is dict:
        if all(type(k) is tuple and len(k) == 2 and isinstance(w, numbers.Number) for k, w in g.items()):
            return "dict_tuple"
        if all(isinstance(d, list) for d in g.values()):
            return "dict_list"
        if all(isinstance(d, dict) and all(isinstance(w, numbers.Number) for w in d.values()) for d in g.values()):
            return "dict_dict"
    if isinstance(g, Iterable) and not isinstance(g, (str, bytes)):
        try:
            seq = list(g)
        except TypeError:
            return None
        if all(type(t) is tuple and len(t) == 2 for t in seq):
            return "tuples2"
        if all(type(t) is tuple and len(t) == 3 for t in seq):
            return "tuples3"
    return None


def _edges_of(g, kind):
    """(vertex symbols, {(u,v): w}) of an edge-dictionary spelling; later duplicates
    overwrite earlier ones, as the nested-dict build in graph.py:1617-1703 does."""
    verts = set()
    edges = {}
    if kind == "dict_tuple":
        for (u, v), w in g.items():
            verts.add(u); verts.add(v)
            edges[(u, v)] = w
    elif kind == "dict_list":
        for u, lst in g.items():
            verts.add(u)
            for v in lst:
                verts.add(v)
                edges[(u, v)] = 1.0
    elif kind == "dict_dict":
        for u, d in g.items():
            verts.add(u)
            for v, w in d.items():
                verts.add(v)
                edges[(u, v)] = w
    elif kind == "tuples2":
        for u, v in g:
            verts.add(u); verts.add(v)
            edges[(u, v)] = 1.0
    elif kind == "tuples3":
        for u, v, w in g:
            verts.add(u); verts.add(v)
            edges[(u, v)] = w
    return verts, edges


class Block:
    """Packed CSR block of a graph list (host, numpy)."""

    def __init__(self, graph_ptr, row_ptr, col_idx, weights, labels, attrs=None, all_adjacency=False):
        self.graph_ptr = np.ascontiguousarray(graph_ptr, dtype=np.int32)
        self.row_ptr = np.ascontiguousarray(row_ptr, dtype=np.int32)
        self.col_idx = np.ascontiguousarray(col_idx, dtype=np.int32)
        self.weights = weights
        self.labels = labels  # list of Python objects (len V) or None
        self.attrs = attrs
        self.all_adjacency = all_adjacency  # every graph came as an adjacency matrix ("auto" -> Floyd-Warshall)
        self.any_adjacency = all_adjacency  # ... or at least one did (pack() refines this for mixed lists)
        self.n_graphs = len(self.graph_ptr) - 1
        self.mode = None  # vertex-set rule the block was packed with: 'wl' | 'sp' | 'wloa' (pack / datasets.read_tu)

    @property
    def n_vertices(self):
        return int(self.graph_ptr[-1])

    @staticmethod
    def concat(a, b):
        """X block followed by Y block (joint relabelling for transform)."""
        va, ea = a.n_vertices, len(a.col_idx)
        gp = np.concatenate([a.graph_ptr, b.graph_ptr[1:] + va])
        rp = np.concatenate([a.row_ptr, b.row_ptr[1:] + ea])
        ci = np.concatenate([a.col_idx, b.col_idx + va])
        w = None
        if a.weights is not None or b.weights is not None:
            wa = a.weights if a.weights is not None else np.ones(ea)
            wb = b.weights if b.weights is not None else np.ones(len(b.col_idx))
            w = np.concatenate([wa, wb])
        if a.labels is None or b.labels is None:
            lab = None
        elif isinstance(a.labels, np.ndarray) and isinstance(b.labels, np.ndarray):
            lab = np.concatenate([a.labels, b.labels])
        else:
            lab = list(a.labels) + list(b.labels)
        at = None if a.attrs is None or b.attrs is None else np.concatenate([a.attrs, b.attrs])
        out = Block(gp, rp, ci, w, lab, at, a.all_adjacency and b.all_adjacency)
        out.any_adjacency = a.any_adjacency or b.any_adjacency
        out.mode = a.mode if a.mode == b.mode else None
        return out

    def require(self, *modes, labels=True):
        """Packed-input fast path of the estimators: the block must carry the vertex set the kernel walks."""
        if self.mode not in modes:
            raise ValueError("this block was packed for another kernel (vertex set %r, needed %s): see "
                             "grakel_b200.datasets.read_tu(kernel=...)" % (self.mode, " or ".join(map(repr, modes))))
        if labels and self.labels is None:
            raise ValueError("Graph does not have any labels for vertices.")
        if self.n_graphs == 0:
            raise ValueError("parsed input is empty")
        return self


def iter_elements(X, len_ok, type_error_msg=None):
    """Yield (index, graph_like, node_labels) for every non-empty element, with the
    reference's element checks (weisfeiler_lehman.py:148-187, shortest_path.py:442-465,
    vertex_histogram.py:86-104): empty elements are skipped with a warning, elements
    of an unacceptable length raise TypeError."""
    if not isinstance(X, Iterable):
        raise TypeError("input must be an iterable\n")
    for idx, x in enumerate(iter(X)):
        if isinstance(x, Graph):
            x = x.as_element()
        is_iter = isinstance(x, Iterable)
        if is_iter:
            x = list(x)
        if not (is_iter and (len(x) == 0 or len_ok(len(x)))):
            raise TypeError(type_error_msg or "each element of X must be either a graph object or a list with at "
                                              "least a graph like object and node labels dict \n")
        if len(x) == 0:
            warnings.warn("Ignoring empty element on index: " + str(idx))
            continue
        yield idx, x[0], (x[1] if len(x) > 1 else None)


def _pack_threads():
    """Worker threads of the CPython-level packer (GRAKEL_B200_PACK_THREADS; default: half the cores, at most 16)."""
    e = os.environ.get("GRAKEL_B200_PACK_THREADS")
    if e:
        return max(1, int(e))
    return max(1, min(16, (os.cpu_count() or 2) // 2))


def _adjacency_array(g):
    if issparse(g):
        A = np.asarray(g.todense())
    else:
        A = np.asarray(g)
    if A.ndim != 2 or A.shape[0] != A.shape[1]:
        raise ValueError("input matrix must be squared")
    return A


_INT_TYPES = {int, np.int64, np.int32}
_NUM_TYPES = {int, float, bool, np.float64, np.float32, np.int64, np.int32}


def _fast_edge_dict(g, L, mode, need_labels, keep_edge_order=False):
    """Vectorised packing of the common spelling {(u, v): w} with integer vertex symbols: every per-edge step
    runs inside C iterators (itertools / map / numpy.fromiter) instead of Python byte code.  Returns
    (n_vertices, src, dst, weights, label list) with the slow path's semantics, or None whenever anything is
    unusual (other symbol types, unlabelled or foreign vertices, ...): the caller then takes the general path,
    which also produces the reference's errors."""
    E = len(g)
    if E == 0 or set(map(type, g)) != {tuple} or set(map(len, g)) != {2}:
        return None
    if not set(map(type, g.values())) <= _NUM_TYPES:
        return None
    if not set(map(type, chain.from_iterable(g))) <= _INT_TYPES:
        return None
    flat = np.fromiter(chain.from_iterable(g), dtype=np.int64, count=2 * E)
    src, dst = flat[0::2], flat[1::2]
    ww = np.fromiter(g.values(), dtype=np.float64, count=E)
    lab_list = None
    if mode == "wl":  # vertex set = label keys; only a contiguous integer range keeps the index arithmetic trivial
        if not L or type(L) is not dict:
            return None
        keys = list(L)
        n = len(keys)
        k0 = keys[0]
        if type(k0) is not int or keys != list(range(k0, k0 + n)):
            return None
        if int(flat.min()) < k0 or int(flat.max()) >= k0 + n:
            return None  # an unlabelled source is skipped, an unlabelled target is a KeyError: general path
        src, dst = src - k0, dst - k0
        lab_list = list(L.values())
    else:  # 'sp' / 'wloa': vertex set = the symbols that occur in an edge, sorted
        sv = np.unique(flat)
        n = len(sv)
        if int(sv[0]) == 0 and int(sv[-1]) == n - 1:
            pass  # already 0..n-1
        else:
            src, dst = np.searchsorted(sv, src), np.searchsorted(sv, dst)
        if need_labels:
            if not L or type(L) is not dict:
                return None
            try:
                lab_list = list(map(L.__getitem__, sv.tolist()))
            except KeyError:
                return None
    order = np.argsort(src, kind="stable") if keep_edge_order else np.lexsort((dst, src))
    return n, src[order], dst[order], ww[order], lab_list


def _lengths_ok(X, len_ok):
    """Element lengths acceptable to the whole-input fast path?  One C-level pass (`map(len, ...)`) instead of a Python
    generator over every element (2-3 ms for 10 000 graphs); the element TYPES are checked by the C packer itself, which
    declines anything that is not an exact list / tuple."""
    try:
        return all(n >= 2 and len_ok(n) for n in set(map(len, X)))
    except TypeError:  # an element without a length: the general loop raises the reference's error
        return False


def pack(X, mode, need_labels=True, len_ok=lambda n: n in (2, 3), want_weights=False,
         fw_zero_is_absent=False, attributes=False, type_error_msg=None, keep_edge_order=False):
    """Pack an iterable of reference-style elements.

    mode = 'wl' : vertex set = the keys of the label dictionary (the reference walks
                  `L[j].keys()`, weisfeiler_lehman.py:234), neighbours = out-edges.
    mode = 'sp' : vertex set = range(n) (adjacency) or the sorted symbols that occur
                  in an edge (dictionary input; graph.py:1613-1631), labels indexed in
                  that order (graph.py:390-394).
    mode = 'wloa': vertex set = the keys of the reference's edge DICTIONARY -- range(n) for
                  adjacency input, the endpoints of the listed edges otherwise; labelled vertices
                  without any edge never reach the histogram
                  (weisfeiler_lehman_optimal_assignment.py:179, 203-209).

    keep_edge_order: a vertex's neighbours stay in the order of the reference's edge dictionary (first listing of
    each edge; ascending columns for adjacency input) instead of ascending vertex id.
    """
    if (_fastpack is not None and type(X) is list and X and not attributes and not fw_zero_is_absent and not keep_edge_order
            and _lengths_ok(X, len_ok)):
        # whole-input fast path: {(u, v): w} graphs with integer symbols, walked with the CPython API on several
        # threads; it declines (None) on anything unusual and the general loop below decides -- and raises -- as before
        res = _fastpack.pack_edge_dicts(X, 0 if mode == "wl" else 1, 1 if need_labels else 0, 1 if want_weights else 0,
                                        _pack_threads())
        if res is not None:
            gp, rp, ci, ww, labs, any_w = res
            if isinstance(labs, bytearray):  # every label is an exact int: int64 values, ids are assigned vectorised
                labs = np.frombuffer(labs, dtype=np.int64)
            out = Block(np.frombuffer(gp, dtype=np.int32), np.frombuffer(rp, dtype=np.int32),
                        np.frombuffer(ci, dtype=np.int32),
                        np.frombuffer(ww, dtype=np.float64) if (want_weights and any_w and ww is not None) else None,
                        labs if need_labels else None, None, False)
            out.mode = mode
            return out
    graph_ptr = [0]
    rp_parts, ci_parts, w_parts = [], [], []
    labels = [] if need_labels else None
    attr_rows = [] if attributes else None
    deg_total = 0
    any_weight = False
    all_adjacency = True
    any_adjacency = False
    for idx, g, L in iter_elements(X, len_ok, type_error_msg):
        base = graph_ptr[-1]
        fast = None
        if type(g) is dict and not attributes and not fw_zero_is_absent:
            fast = _fast_edge_dict(g, L, mode, need_labels, keep_edge_order)
        if fast is not None:
            all_adjacency = False
            verts_n, ii, jj, ww, lab_list = fast
            counts = np.bincount(ii, minlength=verts_n)
            rp_parts.append(deg_total + np.cumsum(counts))
            ci_parts.append(jj + base)
            w_parts.append(ww)
            any_weight = any_weight or bool(np.any(ww != 1.0))
            deg_total += len(ii)
            if need_labels:
                labels.extend(lab_list)
            graph_ptr.append(base + verts_n)
            continue
        kind = classify(g)
        if kind is None:
            raise ValueError("Unsupported input type. For more information check the documentation, concerning "
                             "valid input types for graph type object.")
        base = graph_ptr[-1]
        if kind == "adjacency":
            any_adjacency = True
            A = _adjacency_array(g)
            n = A.shape[0]
            ii, jj = np.nonzero(A > 0)  # graph.py:963 / 1198
            ww = A[ii, jj].astype(np.float64)
            if mode == "wl":
                if not L:
                    raise ValueError("Graph does not have any labels for vertices.")
                keys = list(L.keys())
                if keys == list(range(n)):
                    loc = None
                    verts_n = n
                else:  # labels on a subset / other order: vertex set is the label keys
                    loc = {k: i for i, k in enumerate(keys)}
                    verts_n = len(keys)
                    keep = np.fromiter((int(a) in loc for a in ii), dtype=bool, count=len(ii))
                    ii, jj, ww = ii[keep], jj[keep], ww[keep]
                    try:
                        ii = np.fromiter((loc[int(a)] for a in ii), dtype=np.int64, count=len(ii))
                        jj = np.fromiter((loc[int(b)] for b in jj), dtype=np.int64, count=len(jj))
                    except KeyError as e:
                        raise KeyError(e.args[0])
                    order = np.lexsort((jj, ii))
                    ii, jj, ww = ii[order], jj[order], ww[order]
                lab_list = [L[k] for k in (range(n) if loc is None else keys)]
            else:
                verts_n = n
                if need_labels:
                    if not L:
                        raise ValueError("Graph does not have any labels for vertices.")
                    lab_list = [L[i] for i in range(n)]
            counts = np.bincount(ii, minlength=verts_n)
            rp_parts.append(deg_total + np.cumsum(counts))
            ci_parts.append(jj + base)
            w_parts.append(ww)
            any_weight = any_weight or bool(len(ww) and np.any(ww != 1.0))
            deg_total += len(ii)
        else:
            all_adjacency = False
            verts, edges = _edges_of(g, kind)
            if mode == "wl":
                if not L:
                    raise ValueError("Graph does not have any labels for vertices.")
                keys = list(L.keys())
                loc = {k: i for i, k in enumerate(keys)}
                verts_n = len(keys)
                lab_list = [L[k] for k in keys]
                src, dst, ww = [], [], []
                for (u, v), w in edges.items():
                    iu = loc.get(u)
                    if iu is None:
                        continue  # an unlabelled vertex is never visited by the reference
                    src.append(iu)
                    dst.append(loc[v])  # KeyError like the reference's L[j][n]
                    ww.append(w)
            else:
                if mode == "wloa":  # keys of the edge dictionary = endpoints of listed edges (any order)
                    sv = list(dict.fromkeys(x for e in edges for x in e))
                    if kind == "dict_dict":  # {u: {}} keeps u as a key (graph.py:1660-1667); {u: []} does not
                        sv = list(dict.fromkeys(list(g.keys()) + sv))
                else:
                    sv = sorted(verts)
                loc = {k: i for i, k in enumerate(sv)}
                verts_n = len(sv)
                if need_labels:
                    if not L:
                        raise ValueError("Graph does not have any labels for vertices.")
                    lab_list = [L[k] for k in sv]
                src, dst, ww = [], [], []
                for (u, v), w in edges.items():
                    if fw_zero_is_absent and w == 0:
                        continue  # dictionary -> adjacency -> `dist[dist == 0] = inf` (graph.py:1786)
                    src.append(loc[u])
                    dst.append(loc[v])
                    ww.append(w)
            ii = np.asarray(src, dtype=np.int64)
            jj = np.asarray(dst, dtype=np.int64)
            ww = np.asarray(ww, dtype=np.float64)
            order = np.argsort(ii, kind="stable") if keep_edge_order else np.lexsort((jj, ii))
            ii, jj, ww = ii[order], jj[order], ww[order]
            counts = np.bincount(ii, minlength=verts_n) if len(ii) else np.zeros(verts_n, dtype=np.int64)
            rp_parts.append(deg_total + np.cumsum(counts))
            ci_parts.append(jj + base)
            w_parts.append(ww)
            any_weight = any_weight or bool(len(ww) and np.any(ww != 1.0))
            deg_total += len(ii)
        if need_labels and not attributes:
            labels.extend(lab_list)
        if attributes:
            attr_rows.extend(np.asarray(a, dtype=np.float64).ravel() for a in lab_list)
        graph_ptr.append(base + verts_n)
    if len(graph_ptr) == 1:
        raise ValueError("parsed input is empty")
    row_ptr = np.concatenate([[0]] + rp_parts) if rp_parts else np.zeros(1, dtype=np.int64)
    col_idx = np.concatenate(ci_parts) if ci_parts else np.zeros(0, dtype=np.int64)
    weights = None
    if want_weights and any_weight:
        weights = np.concatenate(w_parts)
    attrs = None
    if attributes:
        attrs = np.asarray(attr_rows, dtype=np.float64)
        if attrs.ndim != 2:
            raise ValueError("node attributes must all have the same length")
    if graph_ptr[-1] >= 2 ** 31 or len(col_idx) >= 2 ** 31:
        raise ValueError("graph block exceeds int32 indexing")
    out = Block(np.asarray(graph_ptr), row_ptr, col_idx, weights, labels, attrs, all_adjacency)
    out.any_adjacency = any_adjacency
    out.mode = mode
    return out


def adjacency_and_labels(g, L=None):
    """The reference's `Graph(g, L, {}, "adjacency").get_adjacency_matrix()` as float64 and, when L is given,
    `get_labels(purpose="adjacency")` in index order (graph.py:912-1053, 1156-1179, 689-772): an adjacency input is taken
    as it is -- every non-zero entry is an edge with its weight, negative ones and self-loops included -- and an edge
    dictionary becomes the matrix over its sorted vertex symbols, every listed symbol a vertex (also one without an
    edge), a later duplicate overwriting an earlier one.  The random walk kernels use this, not pack()."""
    A, order = adjacency_and_order(g)
    labels = None
    if L is not None:
        labels = [L[k] for k in order]
    return A, labels


def adjacency_and_order(g):
    """(the matrix of `adjacency_and_labels`, the vertex symbol of each of its rows): range(n) for an adjacency input,
    the sorted symbols of an edge dictionary."""
    kind = classify(g)
    if kind is None:
        raise ValueError("Unsupported input type. For more information check the documentation, concerning "
                         "valid input types for graph type object.")
    if kind == "adjacency":
        A = np.array(_adjacency_array(g), dtype=np.float64)
        return A, range(A.shape[0])
    verts, edges = _edges_of(g, kind)
    order = sorted(verts)
    loc = {k: i for i, k in enumerate(order)}
    A = np.zeros((len(order), len(order)))
    for (u, v), w in edges.items():
        A[loc[u], loc[v]] = w
    return A, order


def label_ids(labels, known=None, sort_new=True):
    """Dense ids for Python label objects.

    `known` is the fit-time dictionary {label: id}; labels outside it get fresh ids
    >= len(known) (weisfeiler_lehman.py:417-418).  New labels are numbered in sorted
    order like the reference (`sorted(list(distinct_values))`, :204) -- which also
    reproduces its TypeError on mutually incomparable labels -- or in first-seen
    order when `sort_new` is False (ShortestPath only uses labels as dict keys).
    Returns (int32 ids, dictionary of the labels that were new)."""
    known = {} if known is None else known
    if isinstance(labels, np.ndarray) and labels.dtype.kind in "iu":  # integer labels (fast packer, datasets.read_tu)
        lo, hi = (int(labels.min()), int(labels.max())) if len(labels) else (0, 0)
        if len(labels) and hi - lo < (1 << 22):  # small value range: presence table instead of a sort
            present = np.zeros(hi - lo + 1, dtype=bool)
            rel = labels - lo
            present[rel] = True
            uniq = np.flatnonzero(present) + lo
            lut = np.zeros(hi - lo + 1, dtype=np.int32)
            lut[uniq - lo] = np.arange(len(uniq), dtype=np.int32)
            inv = lut[rel]
            first = None
        else:
            uniq, first, inv = np.unique(labels, return_index=True, return_inverse=True)
        if not sort_new:
            if first is None:  # first occurrence of every distinct value
                first = np.full(len(uniq), len(labels), dtype=np.int64)
                np.minimum.at(first, inv, np.arange(len(labels)))
            order = np.argsort(first, kind="stable")
        else:
            order = np.arange(len(uniq))
        fresh, ids_of = {}, np.empty(len(uniq), dtype=np.int32)
        if not known:
            ids_of[order] = np.arange(len(uniq), dtype=np.int32)
            fresh = dict(zip(uniq[order].tolist(), range(len(uniq))))
        else:
            for j in order.tolist():
                l = int(uniq[j])
                if l in known:
                    ids_of[j] = known[l]
                else:
                    ids_of[j] = fresh[l] = len(known) + len(fresh)
        return ids_of[inv].astype(np.int32, copy=False), fresh
    fresh = {}
    seen = set()
    for l in labels:
        if l not in known and l not in seen:
            seen.add(l)
    new = sorted(seen) if sort_new else list(dict.fromkeys(l for l in labels if l in seen))
    base = len(known)
    for i, l in enumerate(new):
        fresh[l] = base + i
    ids = np.fromiter((known[l] if l in known else fresh[l] for l in labels), dtype=np.int32, count=len(labels))
    return ids, fresh
