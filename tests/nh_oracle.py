"""Restatement of NeighborhoodHash (grakel/kernels/neighborhood_hash.py) over packed blocks, for the tests.

Codes are Python ints, so ROT and the XORs follow the reference's unbounded-int arithmetic literally; a vertex whose
code or any out-neighbour's code is None is None.  The count-sensitive hash sorts the neighbour codes
stably by their low `bits` bits and counts runs of equal consecutive values, as the reference's radix sort does, so
the block's rows must list neighbours in the edge dictionary's order.  The level-r intersection counts c_r are a
sparse integer Gram of unary-expanded code histograms (exact), and K = sum(t_r) / R with t_r = c_r / (n_i + n_j - c_r), evaluated
element-wise in float64 the way the reference's built-in `sum` adds floats."""
from collections import Counter

import numpy as np
from scipy import sparse


def rot(n, d, bits):
    """neighborhood_hash.py:367-390."""
    mask = (1 << bits) - 1
    m = d % bits
    if m > 0:
        return (n << m) & mask | ((n & mask) >> (bits - m))
    return n


def hash_level(codes, row_ptr, col_idx, nh_type, bits):
    """One level of neighborhood_hash_simple / neighborhood_hash_count_sensitive (:392-504) over a CSR block."""
    out = []
    for u in range(len(codes)):
        nb = [codes[w] for w in col_idx[row_ptr[u]:row_ptr[u + 1]]]
        if codes[u] is None or any(c is None for c in nb):
            out.append(None)
            continue
        label = rot(codes[u], 1, bits)
        if nh_type == "simple":
            for c in nb:
                label ^= c
        else:
            label ^= radix_sort_rot(nb, bits)
        out.append(label)
    return out


def radix_sort_rot(labels, bits):
    """The count-sensitive term of neighborhood_hash.py:449-504: the neighbour codes sorted stably by their low `bits`
    bits (what its LSD radix sort does; Python's sort is stable), then ROT(value ^ run, run) XOR-ed over the maximal
    runs of equal consecutive values."""
    mask = (1 << bits) - 1
    ordered = sorted(labels, key=lambda c: c & mask)
    result, i = 0, 0
    while i < len(ordered):
        j = i
        while j < len(ordered) and ordered[j] == ordered[i]:
            j += 1
        result ^= rot(ordered[i] ^ (j - i), j - i, bits)
        i = j
    return result


def hash_levels(codes0, row_ptr, col_idx, R, nh_type, bits):
    """[level 0 .. R-1], level 0 = NH(initial codes)."""
    row_ptr = np.asarray(row_ptr).tolist()
    col_idx = np.asarray(col_idx).tolist()
    levels, cur = [], list(codes0)
    for _ in range(R):
        cur = hash_level(cur, row_ptr, col_idx, nh_type, bits)
        levels.append(cur)
    return levels


def as_arrays(level):
    """(uint64 codes with 0 for None, bool valid)."""
    return (np.array([0 if c is None else c for c in level], dtype=np.uint64),
            np.array([c is not None for c in level], dtype=bool))


def intersections(level, graph_ptr):
    """Sparse (N x expanded columns) 0/1 matrix whose Gram is sum_code min(cnt_i, cnt_j) over non-None codes."""
    gp = np.asarray(graph_ptr).tolist()
    col_of, rows, cols = {}, [], []
    for g in range(len(gp) - 1):
        for code, k in Counter(c for c in level[gp[g]:gp[g + 1]] if c is not None).items():
            for t in range(k):
                rows.append(g)
                cols.append(col_of.setdefault((code, t), len(col_of)))
    return sparse.csr_matrix((np.ones(len(rows), dtype=np.int64), (rows, cols)),
                             shape=(len(gp) - 1, max(len(col_of), 1)))


def kernel(levels, graph_ptr, n_fit):
    """fit_transform (n_fit = number of graphs) or transform (rows: graphs n_fit.., columns: graphs ..n_fit)."""
    gp = np.asarray(graph_ptr, dtype=np.int64)
    N = len(gp) - 1
    n = np.diff(gp)
    rows = np.arange(N) if n_fit == N else np.arange(n_fit, N)
    cols = np.arange(n_fit)
    terms = []
    for level in levels:
        S = intersections(level, gp)
        c = np.asarray((S[rows] @ S[cols].T).todense(), dtype=np.int64)
        d = n[rows][:, None] + n[cols][None, :] - c
        terms.append(c.astype(np.float64) / d.astype(np.float64))
    return python_sum(terms) / (1.0 * len(levels))


def python_sum(terms):
    """Element-wise `sum(terms)` as CPython >= 3.12 evaluates a sum of floats started from the int 0: 0 + t_0, then
    Neumaier's compensated addition of every later term, the compensation added at the end when non-zero and finite."""
    s = terms[0] + 0.0
    comp = np.zeros_like(s)
    for x in terms[1:]:
        t = s + x
        comp = comp + np.where(np.abs(s) >= np.abs(x), (s - t) + x, (x - t) + s)
        s = t
    return np.where((comp != 0) & np.isfinite(comp), s + comp, s)
