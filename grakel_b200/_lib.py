"""ctypes binding of libgrakel_b200.so (the C-ABI declared in include/grakel_b200.h).

There is no CPU fallback: if the shared library or an H100 is missing, every
compute entry point raises.  The library is built in-tree by
``__graft_entry__.build()`` (``grakel_b200/csrc/build.sh``).
"""
from __future__ import annotations

import ctypes as C
import os
import threading

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libgrakel_b200.so")

GK_F32, GK_F64 = 0, 1
GK_NORMALIZE, GK_NAN_TO_NUM, GK_GRAM_SIMT, GK_OUT_DEVICE, GK_FULL_TILES, GK_DENSE_ALL = 1, 2, 4, 8, 16, 32
GK_DIST, GK_DIST_GATHER = 64, 128
GK_SP_WITH_LABELS, GK_SP_KEEP_DIST, GK_SP_DIJKSTRA_ORDER = 1, 2, 4
GK_ERR_RANGE, GK_ERR_UNSUPPORTED = -4, -5
GK_GH_LINEAR, GK_GH_GAUSSIAN, GK_GH_BRIDGE = 0, 1, 2
GK_NH_SIMPLE, GK_NH_COUNT_SENSITIVE = 0, 1
GK_RW_CG, GK_RW_SPECTRAL, GK_RW_SERIES = 0, 1, 2
GK_RW_FINITE, GK_RW_EXP, GK_RW_INV = 0, 1, 2
GK_RW_LABELED = 1
GK_PK_ATTR, GK_PK_SQRT, GK_PK_STORE_F32, GK_PK_STORE_INT, GK_PK_NEW_LABELS = 1, 2, 4, 8, 16
GK_PM_LABELS, GK_PM_WL_LABELS = 1, 2
GK_HC_SP = 8
GK_SM_KV_NONE, GK_SM_KV_DIRAC, GK_SM_KE_NONE, GK_SM_KE_DIRAC = 1, 2, 4, 8


class GkStats(C.Structure):
    _fields_ = [
        ("n_graphs", C.c_int64), ("n_vertices", C.c_int64), ("n_edges", C.c_int64),
        ("n_levels", C.c_int64), ("level_dims", C.c_int64 * 64),
        ("n_columns", C.c_int64), ("n_entries", C.c_int64), ("n_dense_columns", C.c_int64),
        ("n_tail_columns", C.c_int64), ("tail_updates", C.c_int64), ("threshold", C.c_int64),
        ("max_count", C.c_int64), ("max_diag", C.c_int64), ("hash_retries", C.c_int64),
        ("gram_path", C.c_int64), ("gemm_tiles", C.c_int64), ("gemm_launches", C.c_int64),
        ("kernel_launches", C.c_int64),
        ("ms_h2d", C.c_float), ("ms_features", C.c_float), ("ms_panel", C.c_float),
        ("ms_gemm", C.c_float), ("ms_tail", C.c_float), ("ms_d2h", C.c_float), ("ms_total", C.c_float),
        ("gemm_elem_bytes", C.c_int64),
        ("ms_hash", C.c_float), ("ms_columns", C.c_float), ("ms_combine", C.c_float),
        ("ms_level_gram", C.c_float * 64), ("nh_order_dependent", C.c_int64),
        ("ms_rw", C.c_float), ("rw_cap_hits", C.c_int64),
        ("ms_propagate", C.c_float), ("pk_near_edge", C.c_int64),
    ]

    def as_dict(self):
        d = {}
        for name, _ in self._fields_:
            v = getattr(self, name)
            d[name] = list(v)[: max(int(self.n_levels), 1)] if name in ("level_dims", "ms_level_gram") else v
        return d


class GrakelB200Error(RuntimeError):
    pass


_P = C.c_void_p
_SYMBOLS = {
    "gk_version": (C.c_int, []),
    "gk_last_error": (C.c_char_p, []),
    "gk_create": (C.c_int, [C.c_int, C.POINTER(_P)]),
    "gk_destroy": (C.c_int, [_P]),
    "gk_sync": (C.c_int, [_P]),
    "gk_pack_csr": (C.c_int, [_P, C.c_int64, _P, _P, _P, _P, _P, _P, C.c_int32]),
    "gk_wl_features": (C.c_int, [_P, C.c_int32, C.POINTER(GkStats)]),
    "gk_sp_features": (C.c_int, [_P, C.c_int32, C.POINTER(GkStats)]),
    "gk_spattr_features": (C.c_int, [_P, C.c_int32, C.POINTER(GkStats)]),
    "gk_wl_sp_features": (C.c_int, [_P, C.c_int32, C.c_int32, C.POINTER(GkStats)]),
    "gk_wl_oa_features": (C.c_int, [_P, C.c_int32, C.POINTER(GkStats)]),
    "gk_gh_features": (C.c_int, [_P, C.c_int32, C.c_double, C.c_int32, C.POINTER(GkStats)]),
    "gk_gh_node_maps": (C.c_int, [_P, C.c_int64, _P]),
    "gk_nh_features": (C.c_int, [_P, C.c_int32, C.c_int32, C.c_int32, _P, _P, C.c_int64, C.c_int32, C.POINTER(GkStats)]),
    "gk_nh_labels": (C.c_int, [_P, C.c_int32, _P, _P]),
    "gk_rw_features": (C.c_int, [_P, C.c_int32, C.c_int32, C.c_double, _P, C.c_int32, _P, _P, _P, _P, _P, _P, C.c_int32,
                                 C.POINTER(GkStats)]),
    "gk_rw_iterations": (C.c_int, [_P, _P]),
    "gk_sm_features": (C.c_int, [_P, C.c_int32, _P, _P, C.c_int32, _P, C.c_int32, _P, C.c_int32, C.POINTER(GkStats)]),
    "gk_sm_counts": (C.c_int, [_P, C.c_int64, C.c_int64, _P]),
    "gk_sm_wl_features": (C.c_int, [_P, C.c_int32, C.c_int32, _P, _P, _P, C.c_int32, _P, C.c_int32,
                                    C.POINTER(GkStats)]),
    "gk_sm_wl_counts": (C.c_int, [_P, C.c_int64, C.c_int64, _P]),
    "gk_sm_hc_features": (C.c_int, [_P, C.c_int32, C.c_int32, _P, _P, _P, C.c_int32, _P, C.c_int32,
                                    C.POINTER(GkStats)]),
    "gk_odd_features": (C.c_int, [_P, C.c_int32, _P, C.c_int32, C.POINTER(GkStats)]),
    "gk_wl_odd_features": (C.c_int, [_P, C.c_int32, C.c_int32, _P, _P, C.c_int32, C.POINTER(GkStats)]),
    "gk_wl_level_sum": (C.c_int, [_P, C.c_int32, C.c_int64, C.c_int64, C.c_int64, C.POINTER(GkStats)]),
    "gk_wl_level_sum_fetch": (C.c_int, [_P, C.c_int32, _P, _P, _P, _P]),
    "gk_core_sum_begin": (C.c_int, [_P, C.c_int64, C.c_int64, C.c_int32]),
    "gk_core_level_add": (C.c_int, [_P, C.c_int32, C.c_int64, C.c_int64, _P, _P, _P, _P, C.POINTER(GkStats)]),
    "gk_odd_info": (C.c_int, [_P, _P]),
    "gk_odd_signatures": (C.c_int, [_P, _P, _P, _P, _P]),
    "gk_selftest_odd_collision": (C.c_int, [_P, C.c_int32]),
    "gk_ml_begin": (C.c_int, [_P, C.c_int32, C.c_double, C.c_double, _P, C.c_int32, C.POINTER(GkStats)]),
    "gk_ml_project": (C.c_int, [_P, _P, C.c_int32, C.c_int32, C.POINTER(GkStats)]),
    "gk_ml_level": (C.c_int, [_P, C.c_int32, _P, C.c_int32, _P, _P, _P, C.POINTER(GkStats)]),
    "gk_ml_finish": (C.c_int, [_P, _P, C.c_int64, _P, C.POINTER(GkStats)]),
    "gk_svmt_solve": (C.c_int, [_P, C.c_int64, _P, _P, C.POINTER(GkStats)]),
    "gk_svmt_draw": (C.c_int, [_P, _P, C.c_int64, _P, C.c_int32, C.c_int32, _P, _P, C.c_int64]),
    "gk_svmt_phi": (C.c_int, [_P, C.c_int32, C.c_int32, _P, _P, C.c_int64, _P, C.c_int64, _P, _P, _P, _P,
                              C.POINTER(GkStats)]),
    "gk_gs_draw": (C.c_int, [_P, _P, C.c_int64, _P, C.c_int32, C.c_int64, _P, _P, C.c_int64, _P]),
    "gk_gs_features": (C.c_int, [_P, C.c_int32, C.c_int64, C.c_int64, _P, _P, _P, C.c_int64, _P, C.c_int64,
                                 C.POINTER(GkStats)]),
    "gk_gs_counts": (C.c_int, [_P, C.c_int64, _P, _P]),
    "gk_pk_features": (C.c_int, [_P, C.c_int32, C.c_double, _P, _P, C.c_int32, C.c_int32, C.c_int64, _P, _P, C.c_int32,
                                 C.POINTER(GkStats)]),
    "gk_pk_hashes": (C.c_int, [_P, C.c_int32, _P, _P]),
    "gk_pm_features": (C.c_int, [_P, C.c_int32, C.c_int32, C.c_int32, _P, _P, _P, C.c_int32, C.c_int32,
                                 C.POINTER(GkStats)]),
    "gk_pm_cells": (C.c_int, [_P, C.c_int32, C.c_int32, _P]),
    "gk_hc_features": (C.c_int, [_P, C.c_int32, C.c_int32, _P, C.c_int32, C.POINTER(GkStats)]),
    "gk_hc_vectors": (C.c_int, [_P, C.c_int32, _P]),
    "gk_selftest_hc_collision": (C.c_int, [_P]),
    "gk_selftest_wl_collision": (C.c_int, [_P, C.c_int32, C.c_int32]),
    "gk_nspd_features": (C.c_int, [_P, C.c_int32, C.c_int32, _P, _P, _P, C.c_int64, _P, _P, _P, C.c_int32, _P, _P, _P,
                                   C.c_int32, _P, C.c_int32, C.POINTER(GkStats)]),
    "gk_nspd_hashes": (C.c_int, [_P, C.c_int32, _P]),
    "gk_selftest_nspd_set_order": (C.c_int, [C.c_int64, _P, _P, _P]),
    "gk_gram": (C.c_int, [_P, C.c_int64, C.c_int32, C.c_int64, C.c_int64, _P, C.c_int32, C.c_int64, _P, _P,
                          C.POINTER(GkStats)]),
    "gk_fetch": (C.c_int, [_P, _P, C.c_int32, C.c_int64]),
    "gk_set_row_map": (C.c_int, [_P, C.c_int64, _P]),
    "gk_wl_labels": (C.c_int, [_P, C.c_int32, _P]),
    "gk_sp_distances": (C.c_int, [_P, C.c_int64, _P]),
    "gk_wl_fit_transform": (C.c_int, [_P, C.c_int64, _P, _P, _P, _P, C.c_int32, C.c_int32, _P, C.c_int32, C.c_int64,
                                      _P, C.POINTER(GkStats)]),
    "gk_wl_gram": (C.c_int, [_P, C.c_int32, C.c_int32, _P, C.c_int32, C.c_int64, _P, C.POINTER(GkStats)]),
    "gk_sp_fit_transform": (C.c_int, [_P, C.c_int64, _P, _P, _P, _P, _P, C.c_int32, C.c_int32, _P, C.c_int32,
                                      C.c_int64, _P, C.POINTER(GkStats)]),
    "gk_event_record": (C.c_int, [_P, C.c_int32]),
    "gk_event_elapsed": (C.c_int, [_P, C.c_int32, C.c_int32, C.POINTER(C.c_float)]),
    "gk_profiler_range": (C.c_int, [C.c_int32]),
    "gk_selftest_gram": (C.c_int, [_P, C.c_int64, C.c_int64, _P, _P, _P]),
    "gk_selftest_live_bytes": (C.c_int, [C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "gk_tu_open": (C.c_int, [C.c_char_p, C.c_char_p, C.c_int32, C.POINTER(_P)]),
    "gk_tu_info": (C.c_int, [_P, C.POINTER(C.c_int64)]),
    "gk_tu_pack": (C.c_int, [_P, C.c_int32, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "gk_tu_fill": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "gk_tu_close": (C.c_int, [_P]),
    "gk_comm_unique_id": (C.c_int, [_P]),
    "gk_comm_init": (C.c_int, [_P, C.c_int32, C.c_int32, _P]),
    "gk_comm_destroy": (C.c_int, [_P]),
    "gk_comm_rows": (C.c_int, [_P, C.c_int64, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "gk_result_device": (C.c_int, [_P, C.POINTER(_P), C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_int64),
                                   C.POINTER(C.c_int32)]),
    "gk_selftest_dist_tiles": (C.c_int, [C.c_int64, C.c_int32, C.c_int32, _P, C.c_int64, C.POINTER(C.c_int64)]),
    "gk_host_alloc": (C.c_int, [C.c_int64, C.POINTER(_P)]),
    "gk_host_free": (C.c_int, [_P, C.c_int64]),
    "gk_selftest_deliver": (C.c_int, [C.c_int32, C.c_int64, C.c_int64, _P, _P, C.c_int32, _P]),
}

_lib = None
_lib_lock = threading.Lock()


def load_library():
    """Load the shared library and bind every symbol of include/grakel_b200.h."""
    global _lib
    with _lib_lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(LIB_PATH):
            raise GrakelB200Error(
                f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(grakel_b200 has no CPU fallback)")
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in _SYMBOLS.items():
            fn = getattr(lib, name)  # AttributeError here = header/library mismatch
            fn.restype = res
            fn.argtypes = args
        _lib = lib
        return lib


def exported_symbols():
    return sorted(_SYMBOLS)


def _ptr(a):
    if a is None:
        return None
    return a.ctypes.data_as(_P)


def _i32(a):
    return np.ascontiguousarray(a, dtype=np.int32)


def nspd_set_order(h0, h1):
    """Host only: iteration order of CPython's set after inserting the distinct pairs with element hashes
    (h0[k], h1[k]) in order k = 0 .. n-1 (the emulation NeighborhoodSubgraphPairwiseDistance runs on the device)."""
    a = np.ascontiguousarray(h0, dtype=np.int64)
    b = np.ascontiguousarray(h1, dtype=np.int64)
    out = np.empty(len(a), dtype=np.int64)
    lib = load_library()
    if lib.gk_selftest_nspd_set_order(len(a), _ptr(a), _ptr(b), _ptr(out)) != 0:
        raise GrakelB200Error(lib.gk_last_error().decode())
    return out


def svmt_draw(rs, sizes, lo, counts):
    """Host only: the index arrays SvmTheta draws with `rs.choice(n, level, replace=False)` for every graph, level
    (lo + column of `counts`, ascending) and sample, concatenated (gk_svmt_draw); `rs` continues after them, its
    gaussian cache untouched."""
    name, key, pos, has_gauss, gauss = rs.get_state()
    key = np.array(key, dtype=np.uint32)
    p = C.c_int32(int(pos))
    sz = _i32(sizes)
    cnt = _i32(counts)
    L = cnt.shape[1]
    levels = lo + np.arange(L)
    n_idx = int(np.sum(cnt * levels * (levels[None, :] <= sz[:, None])))
    idx = np.empty(n_idx, dtype=np.uint8)
    lib = load_library()
    if lib.gk_svmt_draw(_ptr(key), C.byref(p), len(sz), _ptr(sz), int(lo), L, _ptr(cnt), _ptr(idx), n_idx) != 0:
        raise GrakelB200Error(lib.gk_last_error().decode())
    rs.set_state((name, key, p.value, has_gauss, gauss))
    return idx


def gs_draw(rs, sizes, k, n_samples):
    """Host only: GraphletSampling's draws for every graph of `sizes` in order, n_samples each (gk_gs_draw): the size
    rs.randint(min(3, n), min(k, n) + 1) (none when the range is one size) and rs.choice(n, size, replace=False).
    Returns (sizes of the samples u8, their indexes i32 concatenated); `rs` continues after them."""
    name, key, pos, has_gauss, gauss = rs.get_state()
    key = np.array(key, dtype=np.uint32)
    p = C.c_int32(int(pos))
    sz = _i32(sizes)
    cap = int(n_samples) * int(np.minimum(sz, k).sum())
    size = np.empty(len(sz) * int(n_samples), dtype=np.uint8)
    idx = np.empty(max(cap, 1), dtype=np.int32)
    n = C.c_int64()
    lib = load_library()
    if lib.gk_gs_draw(_ptr(key), C.byref(p), len(sz), _ptr(sz), int(k), int(n_samples), _ptr(size), _ptr(idx), cap,
                      C.byref(n)) != 0:
        msg = lib.gk_last_error().decode()
        raise NotImplementedError(msg) if "more than 6" in msg else GrakelB200Error(msg)
    rs.set_state((name, key, p.value, has_gauss, gauss))
    return size, idx[:n.value]


def live_bytes():
    """Tests only: (device, pinned) bytes the library's buffers hold right now, over every engine of the process."""
    dev, pin = C.c_int64(), C.c_int64()
    lib = load_library()
    if lib.gk_selftest_live_bytes(C.byref(dev), C.byref(pin)) != 0:
        raise GrakelB200Error(lib.gk_last_error().decode())
    return dev.value, pin.value


class _HostBlock:
    """Owner of one gk_host_alloc mapping; the ndarray returned to the user keeps it alive through `.base`."""

    def __init__(self, lib, nbytes):
        p = _P()
        if lib.gk_host_alloc(nbytes, C.byref(p)) != 0:
            raise MemoryError("gk_host_alloc(%d) failed: %s" % (nbytes, lib.gk_last_error().decode()))
        self._lib, self.ptr, self.nbytes = lib, p.value, nbytes
        self.__array_interface__ = {"data": (self.ptr, False), "shape": (nbytes,), "typestr": "|u1", "version": 3}

    def __del__(self):
        try:
            if self.ptr:
                self._lib.gk_host_free(self.ptr, self.nbytes)
                self.ptr = None
        except Exception:
            pass


def host_matrix(rows, cols, dtype=np.float64):
    """Fresh C-order (rows, cols) ndarray in a huge-page-backed, pooled host mapping (gk_host_alloc); small
    results come from numpy directly."""
    dt = np.dtype(dtype)
    nbytes = int(rows) * int(cols) * dt.itemsize
    if nbytes < (8 << 20) or os.environ.get("GRAKEL_B200_HOST_ALLOC", "1") == "0":
        return np.empty((rows, cols), dtype=dt)
    block = _HostBlock(load_library(), nbytes)
    return np.asarray(block).view(dt).reshape(rows, cols)


def _gram_out(out, device_ptr, shape, dt):
    """(K, pointer, GK_OUT_DEVICE or 0) of a Gram's output: the raw device pointer `device_ptr`, the caller's host array
    `out`, no matrix (`out=False`) or a fresh host matrix."""
    if device_ptr is not None:
        return None, C.c_void_p(int(device_ptr)), GK_OUT_DEVICE
    if out is False:
        return None, None, 0
    if out is not None:
        assert out.dtype == dt and out.flags.c_contiguous and out.shape == shape
        return out, _ptr(out), 0
    K = host_matrix(*shape, dt)
    return K, _ptr(K), 0


class Engine:
    """One device context (opaque gk_handle + CUDA stream).  Not picklable on
    purpose: estimators keep only host-side state and fetch an engine lazily."""

    def __init__(self, device=None):
        self.lib = load_library()
        if device is None:
            device = int(os.environ.get("GRAKEL_B200_DEVICE", os.environ.get("LOCAL_RANK", "0")))
        self.device = int(device)
        h = _P()
        rc = self.lib.gk_create(self.device, C.byref(h))
        if rc != 0:
            raise GrakelB200Error("gk_create failed: " + self.lib.gk_last_error().decode())
        self.h = h
        self._lock = threading.RLock()

    def close(self):
        """Destroy the handle now (collective when a communicator exists: every rank calls it)."""
        if getattr(self, "h", None):
            self.lib.gk_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != 0:
            msg = self.lib.gk_last_error().decode()
            if rc == GK_ERR_UNSUPPORTED:
                raise NotImplementedError(msg)
            raise GrakelB200Error(f"[{rc}] {msg}")

    # ---- raw entry points -------------------------------------------------
    def pack(self, graph_ptr, row_ptr, col_idx, labels=None, weights=None, attrs=None):
        gp, rp, ci = _i32(graph_ptr), _i32(row_ptr), _i32(col_idx)
        lab = None if labels is None else _i32(labels)
        w = None if weights is None else np.ascontiguousarray(weights, dtype=np.float64)
        at, ad = None, 0
        if attrs is not None:
            at = np.ascontiguousarray(attrs, dtype=np.float64)
            ad = at.shape[1]
        with self._lock:
            self._check(self.lib.gk_pack_csr(self.h, len(gp) - 1, _ptr(gp), _ptr(rp), _ptr(ci), _ptr(lab), _ptr(w),
                                             _ptr(at), ad))
            self.n_graphs = len(gp) - 1

    def set_row_map(self, n_rows, row_of_graph):
        m = None if row_of_graph is None else _i32(row_of_graph)
        with self._lock:
            self._check(self.lib.gk_set_row_map(self.h, int(n_rows), _ptr(m)))

    def wl_features(self, n_iter):
        st = GkStats()
        with self._lock:
            self._check(self.lib.gk_wl_features(self.h, int(n_iter), C.byref(st)))
        return st

    def wl_oa_features(self, n_iter):
        st = GkStats()
        with self._lock:
            self._check(self.lib.gk_wl_oa_features(self.h, int(n_iter), C.byref(st)))
        return st

    def sp_features(self, with_labels=True, keep_dist=False, dijkstra_order=False):
        st = GkStats()
        flags = (GK_SP_WITH_LABELS if with_labels else 0) | (GK_SP_KEEP_DIST if keep_dist else 0)
        flags |= GK_SP_DIJKSTRA_ORDER if dijkstra_order else 0
        with self._lock:
            self._check(self.lib.gk_sp_features(self.h, flags, C.byref(st)))
        return st

    def wl_sp_features(self, n_iter, keep_dist=False, dijkstra_order=True):
        st = GkStats()
        flags = GK_SP_WITH_LABELS | (GK_SP_KEEP_DIST if keep_dist else 0) | (GK_SP_DIJKSTRA_ORDER if dijkstra_order else 0)
        with self._lock:
            self._check(self.lib.gk_wl_sp_features(self.h, int(n_iter), flags, C.byref(st)))
        return st

    def spattr_features(self, dijkstra_order=False):
        st = GkStats()
        with self._lock:
            self._check(self.lib.gk_spattr_features(self.h, GK_SP_DIJKSTRA_ORDER if dijkstra_order else 0, C.byref(st)))
        return st

    def gh_features(self, node_kernel=GK_GH_LINEAR, mu=1.0):
        """GraphHopper node maps and, for the linear node kernel, its feature map (gk_gh_features)."""
        st = GkStats()
        with self._lock:
            self._check(self.lib.gk_gh_features(self.h, int(node_kernel), float(mu), 0, C.byref(st)))
        self.gh_delta = int(st.level_dims[0])
        return st

    def gh_node_maps(self, g, n):
        """Graph g's n x delta x delta node maps M of the last gh_features call."""
        out = np.empty((n, self.gh_delta, self.gh_delta), dtype=np.float64)
        with self._lock:
            self._check(self.lib.gk_gh_node_maps(self.h, int(g), _ptr(out)))
        return out

    def nh_features(self, R, nh_type, bits, code_of_label, label_valid=None):
        """NeighborhoodHash codes of R levels and one expanded count block per level (gk_nh_features).
        `code_of_label[i]` is the initial code of packed label id i, `label_valid[i] == 0` marks it None."""
        codes = np.ascontiguousarray(code_of_label, dtype=np.uint64)
        valid = None if label_valid is None else np.ascontiguousarray(label_valid, dtype=np.uint8)
        st = GkStats()
        with self._lock:
            self._check(self.lib.gk_nh_features(self.h, int(R), int(nh_type), int(bits), _ptr(codes), _ptr(valid),
                                                len(codes), 0, C.byref(st)))
        return st

    def nh_labels(self, level, n_vertices):
        """(codes u64, not-None flags bool) of every packed vertex at NeighborhoodHash level `level`."""
        out = np.empty(n_vertices, dtype=np.uint64)
        valid = np.empty(n_vertices, dtype=np.uint8)
        with self._lock:
            self._check(self.lib.gk_nh_labels(self.h, int(level), _ptr(out), _ptr(valid)))
        return out, valid.astype(bool)

    def rw_features(self, route, fn, lamda, coef=None, values=None, t_row_ptr=None, t_col_idx=None, t_values=None,
                    q=None, w=None, labeled=False):
        """Random walk route of the packed block (gk_rw_features); the next gram() runs it pair by pair."""
        cf = None if coef is None else np.ascontiguousarray(coef, dtype=np.float64)
        f64 = lambda a: None if a is None else np.ascontiguousarray(a, dtype=np.float64)
        vals, tv, qq, ww = f64(values), f64(t_values), f64(q), f64(w)
        trp = None if t_row_ptr is None else _i32(t_row_ptr)
        tci = None if t_col_idx is None else _i32(t_col_idx)
        st = GkStats()
        with self._lock:
            self._check(self.lib.gk_rw_features(self.h, int(route), int(fn), float(lamda), _ptr(cf),
                                                0 if cf is None else len(cf), _ptr(vals), _ptr(trp), _ptr(tci), _ptr(tv),
                                                _ptr(qq), _ptr(ww), GK_RW_LABELED if labeled else 0, C.byref(st)))
        return st

    def sm_features(self, k, lambdas, vtable=None, etable=None, edge_label=None, flags=0):
        """SubgraphMatching records, weight tables and lambdas of the packed block (gk_sm_features); the next gram()
        runs it pair by pair.  vtable / etable: square fp64 tables over the label ids, or None with the matching
        GK_SM_* flag; edge_label[E]: the edge label ids of the packed edges."""
        lam = np.ascontiguousarray(lambdas, dtype=np.float64).ravel()
        vt = None if vtable is None else np.ascontiguousarray(vtable, dtype=np.float64)
        et = None if etable is None else np.ascontiguousarray(etable, dtype=np.float64)
        el = None if edge_label is None else _i32(edge_label)
        st = GkStats()
        with self._lock:
            self._check(self.lib.gk_sm_features(self.h, int(k), _ptr(lam), _ptr(vt), 0 if vt is None else vt.shape[0],
                                                _ptr(et), 0 if et is None else et.shape[0], _ptr(el), int(flags),
                                                C.byref(st)))
        self.sm_k = int(k)
        return st

    def sm_counts(self, n_fit, row):
        """tv [n_fit, k + 1] of the pairs of row `row` of the gram() request with this n_fit."""
        out = np.empty((int(n_fit), self.sm_k + 1), dtype=np.float64)
        with self._lock:
            self._check(self.lib.gk_sm_counts(self.h, int(n_fit), int(row), _ptr(out)))
        return out

    def _sm_level_features(self, fn, n_lv, k, n_iter, level_ids, lambdas, etable, edge_label, flags):
        lam = np.ascontiguousarray(lambdas, dtype=np.float64).ravel()
        et = None if etable is None else np.ascontiguousarray(etable, dtype=np.float64)
        el = None if edge_label is None else _i32(edge_label)
        ids = None if level_ids is None else _i32(level_ids)
        st = GkStats()
        with self._lock:
            self._check(fn(self.h, int(k), int(n_iter), _ptr(ids), _ptr(lam), _ptr(et), 0 if et is None else et.shape[0],
                           _ptr(el), int(flags), C.byref(st)))
        self.sm_k, self.sm_n_lv = int(k), int(n_lv)
        return st

    def sm_wl_features(self, k, n_iter, level_ids, lambdas, etable=None, edge_label=None, flags=0):
        """WeisfeilerLehman over SubgraphMatching (gk_sm_wl_features): level_ids [V, n_iter + 1] the WL class of every
        packed vertex per level (None with GK_SM_KV_NONE); the next gram() returns the level sum in one enumeration."""
        return self._sm_level_features(self.lib.gk_sm_wl_features, int(n_iter) + 1, k, n_iter, level_ids, lambdas,
                                       etable, edge_label, flags)

    def sm_wl_counts(self, n_fit, row):
        """tv [n_fit, n_iter + 1, k + 1] of every level of the pairs of row `row` of the gram() request with this
        n_fit."""
        out = np.empty((int(n_fit), self.sm_n_lv, self.sm_k + 1), dtype=np.float64)
        with self._lock:
            self._check(self.lib.gk_sm_wl_counts(self.h, int(n_fit), int(row), _ptr(out)))
        return out

    def sm_hc_features(self, k, n_iter, level_ids, lambdas, etable=None, edge_label=None, flags=0):
        """HadamardCode over SubgraphMatching (gk_sm_hc_features): level_ids [V, n_iter] the HadamardCode class of
        every packed vertex per level (None with GK_SM_KV_NONE); the next gram() returns the level sum in one
        enumeration."""
        return self._sm_level_features(self.lib.gk_sm_hc_features, n_iter, k, n_iter, level_ids, lambdas, etable,
                                       edge_label, flags)

    def ml_begin(self, L, gamma, heta, phi):
        """MultiscaleLaplacian: adjacency, balls and level-0 features phi [V, dim] of the packed block (gk_ml_begin)."""
        ph = np.ascontiguousarray(phi, dtype=np.float64)
        st = GkStats()
        with self._lock:
            self._check(self.lib.gk_ml_begin(self.h, int(L), float(gamma), float(heta), _ptr(ph), ph.shape[1],
                                             C.byref(st)))
        return st

    def ml_project(self, Q):
        """features <- features Q (gk_ml_project)."""
        q = np.ascontiguousarray(Q, dtype=np.float64)
        st = GkStats()
        with self._lock:
            self._check(self.lib.gk_ml_project(self.h, _ptr(q), q.shape[0], q.shape[1], C.byref(st)))
        return st

    def ml_level(self, level, width, samples=None, samp_rec=None):
        """Vertex records of `level` and the projection against its sample records (gk_ml_level).  Fit: `samples`
        (packed vertex ids) -> (sample records, ns x ns block, stats); transform: `samp_rec` -> (None, None, stats).
        `width` is the current feature width P'."""
        st = GkStats()
        stride = width * width + 1
        if samples is not None:
            ids = _i32(samples)
            ns = len(ids)
            rec = np.empty((ns, stride), dtype=np.float64)
            kss = np.empty((ns, ns), dtype=np.float64)
            with self._lock:
                self._check(self.lib.gk_ml_level(self.h, int(level), _ptr(ids), ns, None, _ptr(rec), _ptr(kss),
                                                 C.byref(st)))
            return rec, kss, st
        sr = np.ascontiguousarray(samp_rec, dtype=np.float64)
        assert sr.shape[1] == stride
        with self._lock:
            self._check(self.lib.gk_ml_level(self.h, int(level), None, sr.shape[0], _ptr(sr), None, None, C.byref(st)))
        return None, None, st

    def ml_finish(self, width, fit_rec=None, want_records=True):
        """Final records of the packed graphs after the fitted ones `fit_rec` (gk_ml_finish): (records or None, stats)."""
        fr = None if fit_rec is None else np.ascontiguousarray(fit_rec, dtype=np.float64)
        out = np.empty((self.n_graphs, width * width + 1), dtype=np.float64) if want_records else None
        st = GkStats()
        with self._lock:
            self._check(self.lib.gk_ml_finish(self.h, _ptr(fr), 0 if fr is None else fr.shape[0], _ptr(out),
                                              C.byref(st)))
        return out, st

    def svmt_solve(self, sizes, adj):
        """SvmTheta: launch the smallest eigenvalues and the one-class SMO of graphs of `sizes` vertices with out-edge
        masks adj [V, 4] u32 (gk_svmt_solve); returns without waiting for them."""
        sz = _i32(sizes)
        a = np.ascontiguousarray(adj, dtype=np.uint32)
        st = GkStats()
        with self._lock:
            self._check(self.lib.gk_svmt_solve(self.h, len(sz), _ptr(sz), _ptr(a), C.byref(st)))
        self._svmt_keep = (sz, a)
        return st

    def svmt_phi(self, lo, counts, idx, fit_phi0=None, details=False):
        """phi [N, L] of the solved graphs from the drawn indexes (gk_svmt_phi), their first level placed after
        `fit_phi0` for gram(); with `details` also (m, alphas, iteration counts).  Returns (phi, details or None, stats)."""
        cnt = _i32(counts)
        ix = np.ascontiguousarray(idx, dtype=np.uint8)
        fp = None if fit_phi0 is None else np.ascontiguousarray(fit_phi0, dtype=np.float64)
        N, L = cnt.shape
        phi = np.empty((N, L), dtype=np.float64)
        det = None
        if details:
            det = (np.empty(N), np.empty(int(np.sum(self._svmt_keep[0]))), np.empty(N, dtype=np.int32))
        st = GkStats()
        with self._lock:
            self._check(self.lib.gk_svmt_phi(self.h, int(lo), L, _ptr(cnt), _ptr(ix), len(ix), _ptr(fp),
                                             0 if fp is None else len(fp), _ptr(phi),
                                             *(_ptr(a) for a in (det or (None, None, None))), C.byref(st)))
        return phi, det, st

    def gs_features(self, k, n_fit, g0, samp_off, samp_size, idx, prior=None):
        """GraphletSampling classes and (graph, class) counts of the packed graphs (gk_gs_features): the samples of the
        graphs g0 .. N-1, the counts `prior` [n, 3] (graph, class code, samples) of the graphs before g0."""
        so = np.ascontiguousarray(samp_off, dtype=np.int64)
        ss = np.ascontiguousarray(samp_size, dtype=np.uint8)
        ix = _i32(idx)
        pr = None if prior is None or len(prior) == 0 else np.ascontiguousarray(prior, dtype=np.int64)
        st = GkStats()
        with self._lock:
            self._check(self.lib.gk_gs_features(self.h, int(k), int(n_fit), int(g0), _ptr(so), _ptr(ss), _ptr(ix),
                                                len(ix), _ptr(pr), 0 if pr is None else len(pr), C.byref(st)))
        return st

    def gs_counts(self):
        """[n, 4] int64 rows (graph, class code, samples, count) of the last gs_features, by graph and code."""
        n = C.c_int64()
        with self._lock:
            self._check(self.lib.gk_gs_counts(self.h, 0, None, C.byref(n)))
            out = np.empty((n.value, 4), dtype=np.int64)
            self._check(self.lib.gk_gs_counts(self.h, n.value, _ptr(out), C.byref(n)))
        return out

    def pk_features(self, t_max, w, u, b, dim, dim_orig, n_fit, t_values, p0=None, flags=0):
        """Propagation bins of t_max levels and their (graph, column) counts (gk_pk_features).  u: [t_max, dim],
        b: [t_max] or [t_max, dim] (GK_PK_ATTR), t_values[E]: the packed CSR's transition entries, p0: [V, dim]."""
        u = np.ascontiguousarray(u, dtype=np.float64)
        b = np.ascontiguousarray(b, dtype=np.float64)
        tv = np.ascontiguousarray(t_values, dtype=np.float64)
        p = None if p0 is None else np.ascontiguousarray(p0, dtype=np.float64)
        st = GkStats()
        with self._lock:
            self._check(self.lib.gk_pk_features(self.h, int(t_max), float(w), _ptr(u), _ptr(b), int(dim), int(dim_orig),
                                                int(n_fit), _ptr(tv), _ptr(p), int(flags), C.byref(st)))
        return st

    def pk_hashes(self, level, n_vertices, width=1):
        """(bins [V, width] fp64, private flags [V] bool) of Propagation level `level`."""
        out = np.empty((n_vertices, width), dtype=np.float64)
        priv = np.empty(n_vertices, dtype=np.uint8)
        with self._lock:
            self._check(self.lib.gk_pk_hashes(self.h, int(level), _ptr(out), _ptr(priv)))
        return out, priv.astype(bool)

    def pm_features(self, L, d, U, n_cols, n_iter=0, flags=0, skip=None):
        """PyramidMatch level blocks (gk_pm_features).  U: [n_sets, V, d] fp64 embeddings, n_cols: [n_sets, N] column
        counts; flags GK_PM_LABELS (packed label ids) or GK_PM_WL_LABELS (WL level s after wl_features(n_iter));
        skip: [V] flags of the vertices without entries, or None."""
        U = np.ascontiguousarray(U, dtype=np.float64)
        nc = np.ascontiguousarray(n_cols, dtype=np.int32)
        sk = None if skip is None else np.ascontiguousarray(skip, dtype=np.uint8)
        st = GkStats()
        with self._lock:
            self._check(self.lib.gk_pm_features(self.h, int(n_iter), int(L), int(d), _ptr(U), _ptr(nc), _ptr(sk),
                                                nc.shape[0], int(flags), C.byref(st)))
        return st

    def pm_cells(self, s, level, n_vertices, d):
        """[V, d] int64 cells of embedding set s at level `level` (-1 past a graph's column count)."""
        out = np.empty((n_vertices, d), dtype=np.int64)
        with self._lock:
            self._check(self.lib.gk_pm_cells(self.h, int(s), int(level), _ptr(out)))
        return out

    def hc_features(self, n_iter, width, skip=None, sp=False, dijkstra_order=False):
        """HadamardCode levels of the packed block (gk_hc_features): n_iter levels of width-`width` vectors, classes per
        level, and the VertexHistogram (sp=False) or ShortestPath (sp=True) block of all levels.  skip: [V] flags of the
        vertices absent from the levels >= 1, or None."""
        sk = None if skip is None else np.ascontiguousarray(skip, dtype=np.uint8)
        flags = (GK_HC_SP if sp else 0) | (GK_SP_DIJKSTRA_ORDER if dijkstra_order else 0)
        st = GkStats()
        with self._lock:
            self._check(self.lib.gk_hc_features(self.h, int(n_iter), int(width), _ptr(sk), flags, C.byref(st)))
        return st

    def hc_vectors(self, level, n_vertices, width):
        """[V, W] int64 vectors of HadamardCode level `level` of the last hc_features call."""
        out = np.empty((n_vertices, width), dtype=np.int64)
        with self._lock:
            self._check(self.lib.gk_hc_vectors(self.h, int(level), _ptr(out)))
        return out

    def selftest_hc_collision(self):
        """Tests only: the next hc_features starts with a degenerate hash, so it must detect collisions and retry."""
        with self._lock:
            self._check(self.lib.gk_selftest_hc_collision(self.h))

    def selftest_wl_collision(self, attempts, from_level=1):
        """Tests only: the next `attempts` WL relabel attempts (each wl_features retry, the asynchronous pass of wl_gram)
        hash the levels >= from_level by (own label, degree) alone, so only the signature verification separates
        classes and every such attempt must detect a collision and be repeated."""
        with self._lock:
            self._check(self.lib.gk_selftest_wl_collision(self.h, int(attempts), int(from_level)))

    def odd_features(self, h, rank):
        """OddSth DAGs, identities and per-bit-plane count tables (gk_odd_features); h < 0: no depth limit."""
        rk = _i32(rank)
        st = GkStats()
        with self._lock:
            self._check(self.lib.gk_odd_features(self.h, int(h), _ptr(rk), 0, C.byref(st)))
        return st

    def wl_odd_features(self, h, n_iter, ids, rank):
        """OddSth over n_iter + 1 WL label sets at once (gk_wl_odd_features): `ids` / `rank` are [n_iter + 1, V], the
        ids of every level above those of the level before."""
        ids, rk = _i32(ids), _i32(rank)
        st = GkStats()
        with self._lock:
            self._check(self.lib.gk_wl_odd_features(self.h, int(h), int(n_iter), _ptr(ids), _ptr(rk), 0, C.byref(st)))
        return st

    def wl_level_sum(self, level, n_fit, row_range=None):
        """Add the K of WL level `level` (the NSPD features just computed) into the device-resident sum."""
        rb, re_ = (0, -1) if row_range is None else row_range
        st = GkStats()
        with self._lock:
            self._check(self.lib.gk_wl_level_sum(self.h, int(level), int(n_fit), int(rb), int(re_), C.byref(st)))
        return st

    def wl_level_sum_fetch(self, rows, cols, normalize=False, xdiag=None, ydiag=None, want_kdiag=False):
        """(K, diagonal of the sum before normalisation or None) of the level sum (gk_wl_level_sum_fetch)."""
        K = host_matrix(rows, cols)
        xd = None if xdiag is None else np.ascontiguousarray(xdiag, dtype=np.float64)
        yd = None if ydiag is None else np.ascontiguousarray(ydiag, dtype=np.float64)
        kd = np.empty(cols, dtype=np.float64) if want_kdiag else None
        flags = (GK_NORMALIZE | GK_NAN_TO_NUM) if normalize else 0
        with self._lock:
            self._check(self.lib.gk_wl_level_sum_fetch(self.h, flags, _ptr(xd), _ptr(yd), _ptr(K), _ptr(kd)))
        return K, kd

    def core_sum_begin(self, n_rows, n_cols, square):
        """Zero the device-resident sum of a CoreFramework fold (gk_core_sum_begin)."""
        with self._lock:
            self._check(self.lib.gk_core_sum_begin(self.h, int(n_rows), int(n_cols), int(bool(square))))

    def core_level_add(self, level, n_fit, rows, cols, n_graphs, want_diag=True, stats=None):
        """Add the K of core level `level` (the base kernel's features just computed; `n_graphs` packed, the first
        `n_fit` its columns) into the sum at rows[j], cols[c] (gk_core_level_add).  Returns (xdiag, ydiag)."""
        rows, cols = _i32(rows), _i32(cols)
        square = n_fit == n_graphs
        xd = np.empty(n_fit, dtype=np.float64) if want_diag else None
        yd = np.empty(n_graphs - n_fit, dtype=np.float64) if (want_diag and not square) else None
        st = stats if stats is not None else GkStats()
        with self._lock:
            self._check(self.lib.gk_core_level_add(self.h, int(level), int(n_fit), len(rows), _ptr(rows), _ptr(cols),
                                                   _ptr(xd), _ptr(yd), C.byref(st)))
        return xd, yd

    def odd_signatures(self):
        """(label id, child offsets, child identity ids, C) of every identity after odd_features."""
        info = np.zeros(3, dtype=np.int64)
        with self._lock:
            self._check(self.lib.gk_odd_info(self.h, _ptr(info)))
            F, nch = int(info[0]), int(info[1])
            label = np.empty(F, dtype=np.int32)
            off = np.empty(F + 1, dtype=np.int64)
            child = np.empty(max(nch, 1), dtype=np.int32)
            Cf = np.empty(F, dtype=np.int32)
            self._check(self.lib.gk_odd_signatures(self.h, _ptr(label), _ptr(off), _ptr(child), _ptr(Cf)))
        return label, off, child[:nch], Cf

    def selftest_odd_collision(self, attempts):
        """Tests only: the next `attempts` identity passes of odd_features hash (label, child count) alone, so each
        must detect a collision and be repeated."""
        with self._lock:
            self._check(self.lib.gk_selftest_odd_collision(self.h, int(attempts)))

    def nspd_features(self, r, d, sym_hash, edge_label, tokens):
        """NeighborhoodSubgraphPairwiseDistance hashes and per-level count tables (gk_nspd_features).  `tokens` is
        the NspdTokens of kernels.py.  Returns (stats, per-graph masks of the distances with pairs)."""
        sh = np.ascontiguousarray(sym_hash, dtype=np.int64)
        el = _i32(edge_label)
        t = tokens
        mask = np.zeros(self.n_graphs, dtype=np.uint64)
        st = GkStats()
        with self._lock:
            self._check(self.lib.gk_nspd_features(
                self.h, int(r), int(d), _ptr(sh), _ptr(el), _ptr(t.tok_rank), int(t.n_labels), _ptr(t.rank_off),
                _ptr(t.rank_bytes), _ptr(t.rank_cp), int(t.n_ranks), _ptr(t.el_off), _ptr(t.el_bytes), _ptr(t.el_cp),
                int(t.n_elabels), _ptr(mask), 0, C.byref(st)))
        return st, mask

    def nspd_hashes(self, radius, n_vertices):
        """H[radius][v] (u32) of every packed vertex after nspd_features."""
        out = np.empty(n_vertices, dtype=np.uint32)
        with self._lock:
            self._check(self.lib.gk_nspd_hashes(self.h, int(radius), _ptr(out)))
        return out

    def rw_iterations(self, rows, cols):
        """CG iterations / series terms of every entry of the last random walk gram() (rows x cols u8)."""
        out = np.empty((rows, cols), dtype=np.uint8)
        with self._lock:
            self._check(self.lib.gk_rw_iterations(self.h, _ptr(out)))
        return out

    def gram(self, n_graphs, n_fit=None, normalize=False, nan_to_num=False, out=None, dtype=np.float64,
             row_range=None, simt=False, full_tiles=False, stats=None, want_diag=True, device_ptr=None, ld=0,
             dense_all=False, dist=False, gather=False):
        """Returns (K, xdiag, ydiag).  K is a fresh C-order numpy array unless
        `out` (host array) or `device_ptr` (raw device pointer) is given."""
        n_fit = n_graphs if n_fit is None else int(n_fit)
        square = n_fit == n_graphs
        rows_total = n_graphs if square else n_graphs - n_fit
        rb, re_ = (0, rows_total) if row_range is None else row_range
        dt = np.dtype(dtype)
        code = GK_F64 if dt == np.float64 else GK_F32
        flags = (GK_NORMALIZE if normalize else 0) | (GK_NAN_TO_NUM if nan_to_num else 0)
        flags |= (GK_GRAM_SIMT if simt else 0) | (GK_FULL_TILES if full_tiles else 0) | (GK_DENSE_ALL if dense_all else 0)
        flags |= (GK_DIST if dist else 0) | (GK_DIST_GATHER if gather else 0)
        K, kptr, oflags = _gram_out(out, device_ptr, (re_ - rb, n_fit), dt)
        flags |= oflags
        xd = np.empty(n_fit, dtype=np.float64) if want_diag else None
        yd = np.empty(n_graphs - n_fit, dtype=np.float64) if (want_diag and not square) else None
        st = stats if stats is not None else GkStats()
        with self._lock:
            self._check(self.lib.gk_gram(self.h, n_fit, flags, rb, re_, kptr, code, int(ld), _ptr(xd), _ptr(yd),
                                         C.byref(st)))
        return K, xd, yd

    # ---- multi-GPU (one process per GPU; collective calls)
    @staticmethod
    def comm_unique_id():
        """128-byte NCCL id created by one rank; hand it to every rank (torch.distributed, MPI, a file ...)."""
        buf = C.create_string_buffer(128)
        lib = load_library()
        if lib.gk_comm_unique_id(buf) != 0:
            raise GrakelB200Error("gk_comm_unique_id: " + lib.gk_last_error().decode())
        return bytes(buf.raw)

    def comm_init(self, nranks, rank, unique_id):
        buf = C.create_string_buffer(bytes(unique_id), 128)
        self._check(self.lib.gk_comm_init(self.h, int(nranks), int(rank), buf))
        self.nranks, self.rank = int(nranks), int(rank)

    def comm_rows(self, n_rows):
        a, b = C.c_int64(), C.c_int64()
        self._check(self.lib.gk_comm_rows(self.h, int(n_rows), C.byref(a), C.byref(b)))
        return a.value, b.value

    def result_device(self):
        """(device pointer, rows, cols, ld, dtype code) of the library-owned result of the last gram()."""
        p, r, c, ld, dt = _P(), C.c_int64(), C.c_int64(), C.c_int64(), C.c_int32()
        self._check(self.lib.gk_result_device(self.h, C.byref(p), C.byref(r), C.byref(c), C.byref(ld), C.byref(dt)))
        return p.value, r.value, c.value, ld.value, dt.value

    def fetch(self, out):
        code = GK_F64 if out.dtype == np.float64 else GK_F32
        self._check(self.lib.gk_fetch(self.h, _ptr(out), code, out.shape[1]))
        return out

    def wl_labels(self, level, n_vertices):
        out = np.empty(n_vertices, dtype=np.int32)
        with self._lock:
            self._check(self.lib.gk_wl_labels(self.h, int(level), _ptr(out)))
        return out

    def sp_distances(self, g, n):
        out = np.empty((n, n), dtype=np.float64)
        with self._lock:
            self._check(self.lib.gk_sp_distances(self.h, int(g), _ptr(out)))
        return out

    def wl_fit_transform_raw(self, graph_ptr, row_ptr, col_idx, labels, n_iter, out, normalize=False):
        """One C call, host buffers in / host buffer out (the e2e path of bench.py)."""
        st = GkStats()
        code = GK_F64 if out.dtype == np.float64 else GK_F32
        flags = (GK_NORMALIZE | GK_NAN_TO_NUM) if normalize else 0
        with self._lock:
            self._check(self.lib.gk_wl_fit_transform(self.h, len(graph_ptr) - 1, _ptr(graph_ptr), _ptr(row_ptr),
                                                     _ptr(col_idx), _ptr(labels), int(n_iter), flags, _ptr(out), code,
                                                     out.shape[1], None, C.byref(st)))
        return st

    def wl_gram(self, n_iter, out=None, dtype=np.float64, device_ptr=None, ld=0, dense_all=False, want_diag=False,
                stats=None):
        """WL features + square Gram of the packed block in ONE C call (gk_wl_gram): the asynchronous pass -- one host
        synchronisation, head/tail decision on the device -- when it applies, else gk_wl_features + gk_gram.
        Returns (K, xdiag, stats); `out` / `device_ptr` as in gram()."""
        n = self.n_graphs
        dt = np.dtype(dtype)
        code = GK_F64 if dt == np.float64 else GK_F32
        flags = GK_DENSE_ALL if dense_all else 0
        K, kptr, oflags = _gram_out(out, device_ptr, (n, n), dt)
        flags |= oflags
        xd = np.empty(n, dtype=np.float64) if want_diag else None
        st = stats if stats is not None else GkStats()
        with self._lock:
            self._check(self.lib.gk_wl_gram(self.h, int(n_iter), flags, kptr, code, int(ld), _ptr(xd), C.byref(st)))
        return K, xd, st

    def selftest_gram(self, counts):
        counts = np.ascontiguousarray(counts, dtype=np.uint16)
        n, d = counts.shape
        a = np.empty((n, n), dtype=np.float64)
        b = np.empty((n, n), dtype=np.float64)
        with self._lock:
            self._check(self.lib.gk_selftest_gram(self.h, n, d, _ptr(counts), _ptr(a), _ptr(b)))
        return a, b

    def selftest_deliver(self, src, mode=0, diag=None, nan_to_num=False):
        """Host-only: fp32 matrix -> float64 through the delivery code of gk_gram (no device work).  mode 0: upper
        triangle as fp32, 1: all rows, 2: all rows + normalisation, 3: upper triangle band-packed as u16."""
        src = np.ascontiguousarray(src, dtype=np.float32)
        rows, cols = src.shape
        dst = np.full((rows, cols), np.nan)
        dg = None if diag is None else np.ascontiguousarray(diag, dtype=np.float64)
        self._check(self.lib.gk_selftest_deliver(int(mode), rows, cols, _ptr(src), _ptr(dg), 1 if nan_to_num else 0, _ptr(dst)))
        return dst

    def event_record(self, slot):
        self._check(self.lib.gk_event_record(self.h, slot))

    def event_elapsed(self, a, b):
        ms = C.c_float()
        self._check(self.lib.gk_event_elapsed(self.h, a, b, C.byref(ms)))
        return ms.value

    def profiler_range(self, on):
        self._check(self.lib.gk_profiler_range(1 if on else 0))

    def sync(self):
        self._check(self.lib.gk_sync(self.h))


_engines = {}
_engines_lock = threading.Lock()
_default_device = None


def set_default_device(device):
    """Device ordinal new estimator runs use (default: GRAKEL_B200_DEVICE, else LOCAL_RANK, else 0)."""
    global _default_device
    _default_device = None if device is None else int(device)


def default_device():
    if _default_device is not None:
        return _default_device
    return int(os.environ.get("GRAKEL_B200_DEVICE", os.environ.get("LOCAL_RANK", "0")))


def get_engine(device=None):
    """The process-wide engine of a device (bench / tools / tests that drive the C-ABI step by step)."""
    if device is None:
        device = default_device()
    with _engines_lock:
        e = _engines.get(device)
        if e is None:
            e = Engine(device)
            _engines[device] = e
        return e


class _EnginePool:
    """Engines of one device handed out to estimator runs: a run holds one engine (one handle + stream) for its
    pack -> features -> gram sequence, so estimators used from several Python threads (sklearn's threading
    backend) run concurrently on separate streams instead of serialising on one handle.  At most
    GRAKEL_B200_MAX_ENGINES (default 4) engines per device; further threads wait for a free one."""

    def __init__(self, device):
        self.device = device
        self.free = []
        self.count = 0
        self.cv = threading.Condition()
        self.limit = max(1, int(os.environ.get("GRAKEL_B200_MAX_ENGINES", "4")))

    def acquire(self):
        with self.cv:
            while True:
                if self.free:
                    return self.free.pop()
                if self.count < self.limit:
                    self.count += 1
                    break
                self.cv.wait()
        try:
            # the first engine of the pool is the process-wide one, so step-by-step users share its buffers
            return get_engine(self.device) if self.count == 1 else Engine(self.device)
        except Exception:
            with self.cv:
                self.count -= 1
                self.cv.notify()
            raise

    def release(self, eng):
        with self.cv:
            self.free.append(eng)
            self.cv.notify()


_pools = {}


class engine:
    """`with engine(device) as eng:` -- exclusive use of one engine of the device for the duration."""

    def __init__(self, device=None):
        self.device = default_device() if device is None else int(device)
        self.eng = None

    def __enter__(self):
        with _engines_lock:
            pool = _pools.get(self.device)
            if pool is None:
                pool = _pools[self.device] = _EnginePool(self.device)
        self.pool = pool
        self.eng = pool.acquire()
        self.eng._lock.acquire()
        return self.eng

    def __exit__(self, *exc):
        self.eng._lock.release()
        self.pool.release(self.eng)
        return False
