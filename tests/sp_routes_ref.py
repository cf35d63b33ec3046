"""Float64 restatement of the shortest-path feature block, the dispatch rule of sp_features_impl, and the cases of
test_gpu_sp_routes.py.

Reference: the APSP of every packed graph in the order the reference's algorithm sums paths (scipy BFS for unit
weights, the oracle's k-ordered fp64 Floyd-Warshall, the oracle's Dijkstra), then one feature per (graph, l(u), l(v),
bit pattern of d(u, v)) over ordered pairs u != v at finite distance, counted with np.unique, and K = Phi Phi^T in
int64.  WL-SP takes its level labels from blockref.wl_levels, HC-SP from the level classes of hc_oracle; either way
the ids are made level-unique, so one feature block holds every level."""
import numpy as np
from scipy.sparse import csr_matrix
from scipy.sparse.csgraph import shortest_path

import blockref
import hc_oracle
from grakel_b200.packing import pack
from oracle.gk_oracle import OGraph, _looks_like_adjacency

# ---------------------------------------------------------------- dispatch rule of sp_features_impl (api.cu)
SMEM_DIST_MAX = 160 * 1024    # fp64 distance matrices up to this size stay in shared memory: n <= 143
LOCAL_SLOTS = 2048            # SP_LOCAL_SLOTS: the CTA table of the BFS and Floyd-Warshall kernels
DIRECT_MAX_LABELS = 11        # SP_DIRECT_MAX_LABELS
DICT_CAP0 = 1 << 16           # starting feature dictionary (grown when more than half full)
DKEY_CAP0 = 1 << 18           # starting distance dictionary of real mode
DKEY_CAP_MAX = 1 << 24        # the 24-bit distance field of a real-mode feature key

ROUTES = (
    "bfs_w1", "bfs_w2", "bfs_w4", "bfs_w8",          # bitmask BFS word classes (n <= 64 / 128 / 256 / 512)
    "bfs_t32", "bfs_t64", "bfs_t128",                # BFS thread count from the class's largest graph
    "bfs_direct", "bfs_past_dcap",                   # direct (ls, lv, level) table; a level beyond dcap
    "bfs_hashed", "bfs_hashed_fallthrough",          # hashed CTA table; more keys than it holds
    "fw_u16_global",                                 # unit weights, n > 512
    "fw_f64_shared", "fw_f64_global",                # integer weights, n <= 143 / n >= 144
    "real_switch",                                   # a non-integer distance or one >= 2^24
    "real_fw_shared", "real_fw_global", "real_dj_shared", "real_dj_global",
    "dict_regrow", "ft_regrow", "dkey_regrow",       # the attempt loop
    "keep_dist",                                     # GK_SP_KEEP_DIST
)


def dcap(L):
    return LOCAL_SLOTS // (L * L)


def word_class(n):
    return 0 if n <= 64 else 1 if n <= 128 else 2 if n <= 256 else 3


def route(n, weight_kind, L, order="fw"):
    """Routes one graph of n vertices takes; weight_kind 'unit' | 'int' | 'real', L = total label count."""
    if n <= 0:
        return set()
    if weight_kind == "unit":
        if n <= 512:
            return {"bfs_w%d" % (1 << word_class(n)), "bfs_direct" if L <= DIRECT_MAX_LABELS else "bfs_hashed"}
        return {"fw_u16_global"}
    place = "shared" if n * n * 8 <= SMEM_DIST_MAX else "global"
    if weight_kind == "int":
        return {"fw_f64_" + place}
    return {"real_switch", ("real_dj_" if order == "dijkstra" else "real_fw_") + place}


def call_routes(sizes, weight_kind, L, order="fw"):
    """Routes of one call: every graph's, plus the BFS thread count, which each word class takes from its largest
    graph."""
    out = set()
    cls_max = {}
    for n in sizes:
        out |= route(int(n), weight_kind, L, order)
        if weight_kind == "unit" and 0 < n <= 512:
            c = word_class(n)
            cls_max[c] = max(cls_max.get(c, 0), int(n))
    for m in cls_max.values():
        out.add("bfs_t%d" % (32 if m <= 32 else 64 if m <= 64 else 128))
    return out


def ft_cap0(V, n_pass):
    x = max(V, 1024) * 16 * min(n_pass, 4)
    return max(1 << (x - 1).bit_length(), 1 << 20)


# ---------------------------------------------------------------- reference
def weight_kind(block):
    w = block.weights
    if w is None or np.all(w == 1.0):
        return "unit"
    return "int" if np.all(w == np.rint(w)) else "real"


def graph_csr(block, g):
    v0, v1 = int(block.graph_ptr[g]), int(block.graph_ptr[g + 1])
    e0, e1 = int(block.row_ptr[v0]), int(block.row_ptr[v1])
    rp = block.row_ptr[v0:v1 + 1].astype(np.int64) - e0
    ci = block.col_idx[e0:e1].astype(np.int64) - v0
    w = np.ones(e1 - e0) if block.weights is None else np.asarray(block.weights[e0:e1], dtype=np.float64)
    return v1 - v0, rp, ci, w


def apsp(block, g, order):
    """order: 'unit' (BFS), 'fw' (k-ordered fp64 Floyd-Warshall) or 'dijkstra' (the reference's heap Dijkstra)."""
    n, rp, ci, w = graph_csr(block, g)
    if n == 0:
        return np.zeros((0, 0))
    if order == "unit":
        return shortest_path(csr_matrix((np.ones(len(ci)), ci, rp), shape=(n, n)), directed=True, unweighted=True)
    src = np.repeat(np.arange(n), np.diff(rp))
    if order == "fw":
        A = np.zeros((n, n))
        A[src, ci] = w
        return OGraph(A, {}).floyd_warshall()
    ed = {u: {} for u in range(n)}
    for u, v, x in zip(src.tolist(), ci.tolist(), w.tolist()):
        ed[u][v] = x
    return OGraph(ed, {}).dijkstra_all()


def dense_ids(labels):
    enum = {}
    return np.fromiter((enum.setdefault(x, len(enum)) for x in (labels.tolist() if isinstance(labels, np.ndarray)
                                                                 else labels)), dtype=np.int64, count=len(labels))


def level_labels(levels):
    """Level-unique ids: level i's ids shifted past every id of the levels before it."""
    out, base = [], 0
    for lab in levels:
        out.append(np.asarray(lab, dtype=np.int64) + base)
        base += int(lab.max()) + 1 if len(lab) else 0
    return out


def features(block, label_sets, order):
    """Phi (int64, graphs x distinct features) and what the dispatch depends on."""
    N = block.n_graphs
    parts, dists = [], []
    info = {"depth": 0, "max_local": 0, "max_dist": 0.0, "nonint": False}
    for g in range(N):
        D = apsp(block, g, order)
        dists.append(D)
        n = D.shape[0]
        u, v = np.nonzero(np.isfinite(D) & ~np.eye(n, dtype=bool))
        d = np.ascontiguousarray(D[u, v], dtype=np.float64)
        if len(d):
            info["depth"] = max(info["depth"], int(d.max()) if order == "unit" else 0)
            info["max_dist"] = max(info["max_dist"], float(d.max()))
            info["nonint"] |= bool(np.any(d != np.rint(d)))
        v0 = int(block.graph_ptr[g])
        for lab in label_sets:
            lu = lab[v0 + u] if lab is not None else np.zeros(len(u), dtype=np.int64)
            lv = lab[v0 + v] if lab is not None else np.zeros(len(u), dtype=np.int64)
            R = np.stack([np.full(len(u), g, dtype=np.int64), lu, lv, d.view(np.int64)], axis=1)
            info["max_local"] = max(info["max_local"], len(np.unique(R[:, 1:], axis=0)) if len(R) else 0)
            parts.append(R)
    R = np.concatenate(parts) if parts else np.zeros((0, 4), dtype=np.int64)
    keys, col = np.unique(R[:, 1:], axis=0, return_inverse=True)
    gc, cnt = np.unique(np.stack([R[:, 0], col.reshape(-1)], axis=1), axis=0, return_counts=True)
    Phi = csr_matrix((cnt.astype(np.int64), (gc[:, 0], gc[:, 1])), shape=(N, max(len(keys), 1)), dtype=np.int64)
    info.update(n_columns=len(keys), n_pairs=len(gc), n_lengths=len(np.unique(R[:, 3])), dists=dists)
    return Phi, info


def gram(Phi):
    return np.asarray((Phi @ Phi.T).toarray(), dtype=np.int64)


def normalized(K, xdiag, ydiag):
    with np.errstate(divide="ignore", invalid="ignore"):
        return K / np.sqrt(np.outer(ydiag.astype(np.float64), xdiag.astype(np.float64)))


def path_order(X, block, algorithm_type="auto", wl=False):
    """The reference's path-sum order for real weights: Dijkstra for edge dictionaries under "auto" (and always for
    the edge dictionaries WL hands its base kernel), Floyd-Warshall for adjacency input."""
    kind = weight_kind(block)
    if kind == "unit":
        return "unit"
    if kind == "int" or algorithm_type == "floyd_warshall":
        return "fw"
    if wl or algorithm_type == "dijkstra" or not _looks_like_adjacency(X[0][0]):
        return "dijkstra"
    return "fw"


def prepare(X, Y=None, with_labels=True, algorithm_type="auto", wl_iter=None, hc_iter=None):
    """The packed block of X followed by Y, the label ids of every level, and the path-sum order.  wl_iter / hc_iter:
    number of levels of WL-SP / HC-SP (the estimators' n_iter)."""
    full = list(X) + (list(Y) if Y is not None else [])
    nx = len(X)
    if wl_iter is not None:
        block = pack(full, "wl", want_weights=True)
        label_sets = level_labels(blockref.wl_levels(block, dense_ids(block.labels), wl_iter - 1))
        order = path_order(full, block, wl=True)
    else:
        block = pack(full, "sp", need_labels=with_labels or hc_iter is not None, want_weights=True,
                     len_ok=lambda n: n in (2, 3) or (n == 1 and not with_labels),
                     fw_zero_is_absent=algorithm_type == "floyd_warshall")
        order = path_order(full, block, algorithm_type)
        if hc_iter is not None:
            enum = hc_oracle.enumerate_labels(x[1] for x in X)
            enum = hc_oracle.enumerate_labels((y[1] for y in full[nx:]), enum)
            levels = []
            for lv in hc_oracle.levels(full, hc_iter, enum):
                rows = np.concatenate([np.array(list(d.values()), dtype=np.int64).reshape(len(d), -1) for d in lv])
                levels.append(np.unique(rows, axis=0, return_inverse=True)[1].reshape(-1))
            label_sets = level_labels(levels)
        else:
            label_sets = [dense_ids(block.labels)] if with_labels else [None]
    return {"block": block, "label_sets": label_sets, "order": order, "nx": len(X), "has_y": Y is not None}


def reference(X, Y=None, with_labels=True, algorithm_type="auto", wl_iter=None, hc_iter=None):
    """K of fit_transform(X) (int64), K of transform(Y) when Y is given, the diagonals, and the feature info of the
    joint call and of the fit call alone."""
    out = prepare(X, Y, with_labels, algorithm_type, wl_iter, hc_iter)
    block, label_sets, order, nx = out["block"], out["label_sets"], out["order"], out["nx"]
    Phi, info = features(block, label_sets, order)
    K = gram(Phi)
    diag = np.diagonal(K).copy()
    out.update(K=K[:nx, :nx], xdiag=diag[:nx], full=K, info=info)
    if Y is not None:
        out.update(Kt=K[nx:, :nx], ydiag=diag[nx:], fit_info=_fit_info(block, label_sets, order, nx))
    else:
        out["fit_info"] = info
    return out


def _sub_block(block, nx):
    from grakel_b200.packing import Block
    gp = block.graph_ptr[:nx + 1]
    V = int(gp[-1])
    E = int(block.row_ptr[V])
    return Block(gp, block.row_ptr[:V + 1], block.col_idx[:E], None if block.weights is None else block.weights[:E],
                 None)


def _fit_info(block, label_sets, order, nx):
    V = int(block.graph_ptr[nx])
    return features(_sub_block(block, nx), [None if s is None else s[:V] for s in label_sets], order)[1]


def n_labels(label_sets, V=None):
    """Total label count the device sees over the first V vertices: the sum of the levels' distinct labels
    (level_base[n_pass]), the packed ids' count for plain SP, 1 without labels."""
    if label_sets[0] is None:
        return 1
    return int(sum(len(np.unique(s[:V])) for s in label_sets))


# ---------------------------------------------------------------- inputs
def graph(rs, n, deg=3.0, directed=False, weights=None, L=7, lab0=0, loops=0, isolated=0, path=False, cycle=False,
          as_dict=False, wmax=5):
    """[adjacency or {(u, v): w}, labels].  Every label 0 .. L-1 occurs when n >= L (ids offset by lab0)."""
    pairs = []
    live = n - isolated
    if path:
        pairs += [(i, i + 1) for i in range(live - 1)]
    if cycle:
        pairs += [(i, (i + 1) % live) for i in range(live)] if live > 1 else []
    m = int(deg * n / (1 if directed else 2))
    if live > 1 and m:
        a, b = rs.randint(0, live, m), rs.randint(0, live, m)
        pairs += [(int(x), int(y)) for x, y in zip(a, b) if x != y]
    if loops:
        pairs += [(int(x), int(x)) for x in rs.randint(0, max(live, 1), loops)]
    if not directed:
        pairs += [(v, u) for u, v in pairs]
    ed = {}
    for u, v in pairs:
        if (u, v) in ed:
            continue
        if weights is None:
            w = 1.0
        elif weights == "int":
            w = float(rs.randint(1, wmax + 1))
        else:
            w = float(rs.rand() + 0.05)
        ed[(u, v)] = w
        if not directed and (v, u) not in ed:
            ed[(v, u)] = w
    lab = np.concatenate([np.arange(min(L, n)), rs.randint(0, L, max(n - L, 0))]) + lab0
    rs.shuffle(lab)
    labels = {i: int(x) for i, x in enumerate(lab)}
    if as_dict:
        return [ed, labels]
    A = np.zeros((n, n))
    for (u, v), w in ed.items():
        A[u, v] = w
    return [A, labels]


def gset(seed, sizes, **kw):
    rs = np.random.RandomState(seed)
    return [graph(rs, int(n), **kw) for n in sizes]


def path_graph(n, L, weights=None):
    A = np.zeros((n, n))
    i = np.arange(n - 1)
    A[i, i + 1] = A[i + 1, i] = 1.0 if weights is None else weights
    return [A, {v: v % L for v in range(n)}]


def two_edge_path(w1, w2):
    A = np.zeros((3, 3))
    A[0, 1] = A[1, 0] = float(w1)
    A[1, 2] = A[2, 1] = float(w2)
    return [A, {0: 0, 1: 1, 2: 0}]


def _case(cid, X, Y=None, kind="unit", est="sp", expect=(), keep=True, **kw):
    return dict(id=cid, X=X, Y=Y, kind=kind, est=est, expect=set(expect), keep=keep, **kw)


def cases():
    """Each case: the estimator it goes through (sp / wlsp / hcsp), its inputs, and the routes it is meant to
    reach.  The data-dependent routes (a level past dcap, a full CTA table, regrowth) are asserted from the reference
    when the case runs; the size-dependent ones are checked here by test_sp_routes_ref.py."""
    C = []
    unseen = lambda seed, sizes, **kw: gset(seed, sizes, lab0=5, **kw)  # labels 5 .. 11: 7 .. 11 are unseen
    for n in (1, 2, 32, 33, 64, 65, 128, 129, 256, 257, 511, 512):
        X = gset(n, [n, max(1, n // 2), n], directed=n % 2 == 1, loops=2 if n > 2 else 0, isolated=1 if n > 8 else 0)
        C.append(_case("bfs_n%d" % n, X, unseen(n + 1, [max(1, n // 3), n]), expect=()))
    C.append(_case("bfs_mixed_classes", gset(3, [40, 100, 200, 400, 20, 500, 64, 65]),
                   gset(4, [30, 130, 300], lab0=3)))
    # direct table around dcap: L = 11 (dcap 16) on 40-vertex paths, L = 3 (dcap 227) on a 300-vertex path
    C.append(_case("direct_L11_paths", [path_graph(40, 11), path_graph(17, 11), path_graph(18, 11)] +
                   gset(5, [30], L=11), gset(6, [20], L=11), expect={"bfs_past_dcap"}))
    C.append(_case("direct_L3_path300", [path_graph(300, 3), path_graph(228, 3)] + gset(7, [100], L=3),
                   gset(8, [50], L=3), expect={"bfs_past_dcap"}))
    C.append(_case("hashed_L12", gset(9, [50, 120, 250, 500], L=12), gset(10, [60], L=12, lab0=2)))
    C.append(_case("no_labels", gset(11, [300, 40, 129], directed=True), gset(12, [70]), with_labels=False))
    C.append(_case("hashed_fallthrough_400_labels", gset(13, [512, 512, 480], L=400, deg=2.0), None,
                   expect={"bfs_hashed_fallthrough"}))
    # unit-weight Floyd-Warshall in global memory: disconnected parts, directed edges
    C.append(_case("fw_u16_global", gset(14, [513, 700], directed=True, isolated=30, deg=2.5) + gset(15, [40]),
                   gset(16, [520], lab0=2)))
    # integer weights: fp64 Floyd-Warshall in shared memory (n = 143) and in global memory (n = 144)
    C.append(_case("fw_f64_143_144", gset(17, [143, 144, 20], directed=True, weights="int"),
                   gset(18, [144, 10], weights="int", lab0=3), kind="int"))
    C.append(_case("int_sum_2p24_minus_1", [two_edge_path(1 << 23, (1 << 23) - 1), path_graph(4, 2, weights=2.0)],
                   kind="int"))
    C.append(_case("int_sum_2p24_real_mode", [two_edge_path(1 << 23, 1 << 23), path_graph(4, 2, weights=3.0)],
                   kind="int", expect={"real_switch", "real_fw_shared"}))
    # real weights, both path-sum orders, both sides of the shared-memory limit, directed
    C.append(_case("real_fw_143_150", gset(19, [143, 150, 30], directed=True, weights="real"),
                   gset(20, [145, 12], directed=True, weights="real", lab0=2), kind="real"))
    C.append(_case("real_dj_143_150", gset(21, [143, 150, 30], directed=True, weights="real", cycle=True,
                                            as_dict=True),
                   gset(22, [144, 12], directed=True, weights="real", cycle=True, as_dict=True, lab0=2),
                   kind="real"))
    C.append(_case("wlsp_real_150", gset(23, [150, 60, 30], directed=True, weights="real"),
                   gset(24, [40], directed=True, weights="real"), kind="real", est="wlsp", n_iter=3))
    C.append(_case("wlsp_hashed_bfs", gset(25, [40, 100, 300], L=5), gset(26, [80], L=5), est="wlsp", n_iter=3))
    C.append(_case("wlsp_u16_global", gset(27, [600, 50], directed=True, deg=2.0), None, est="wlsp", n_iter=2))
    C.append(_case("hcsp_int_150", gset(28, [150, 90, 40], weights="int"), gset(29, [150], weights="int"),
                   kind="int", est="hcsp", n_iter=2))
    # regrowth of the feature dictionary and the (graph, column) table: 200 labels make nearly every pair of a graph
    # a feature of its own (about 1.2 million (graph, column) pairs against a starting table of 2^20)
    C.append(_case("sp_regrow", gset(30, [64] * 300, deg=3.0, L=200), None, expect={"dict_regrow", "ft_regrow"}))
    # real mode: more distinct lengths than the distance dictionary's starting size
    C.append(_case("real_dkey_regrow", gset(31, [40] * 300, directed=True, weights="real", cycle=True, deg=2.0,
                                            L=3), None,
                   kind="real", expect={"dkey_regrow", "dict_regrow"}, fresh=True))
    C.append(_case("real_dkey_regrow_small_cap", gset(32, [20] * 10, directed=True, weights="real", cycle=True),
                   gset(33, [20] * 2, directed=True, weights="real", cycle=True), kind="real",
                   expect={"dkey_regrow"}, env={"GRAKEL_B200_SP_DKEY_CAP": "1024"}, dkey0=1024))
    return C


def case_args(c):
    return dict(with_labels=c.get("with_labels", True), algorithm_type=c.get("algorithm_type", "auto"),
                wl_iter=c.get("n_iter") if c["est"] == "wlsp" else None,
                hc_iter=c.get("n_iter") if c["est"] == "hcsp" else None)


def _fit_labels(r):
    return n_labels(r["label_sets"], int(r["block"].graph_ptr[r["nx"]]))


def case_routes(c, r):
    """Size-dependent routes of a case from prepare() / reference() r: its fit call and, with Y, the joint call."""
    block, nx = r["block"], r["nx"]
    sizes = np.diff(block.graph_ptr)
    order = "dijkstra" if r["order"] == "dijkstra" else "fw"
    out = call_routes(sizes[:nx], c["kind"], _fit_labels(r), order)
    if r["has_y"]:
        out |= call_routes(sizes, c["kind"], n_labels(r["label_sets"]), order)
    if c["est"] == "sp" and c["keep"]:
        out.add("keep_dist")
    return out


def data_routes(c, r):
    """Data-dependent routes the reference r shows the fit call reaches."""
    fit, nx = r["fit_info"], r["nx"]
    L = _fit_labels(r)
    out = set()
    if c["kind"] == "unit" and L <= DIRECT_MAX_LABELS and fit["depth"] > dcap(L):
        out.add("bfs_past_dcap")
    if c["kind"] == "unit" and L > DIRECT_MAX_LABELS and fit["max_local"] > LOCAL_SLOTS:
        out.add("bfs_hashed_fallthrough")
    if c["kind"] == "int" and fit["max_dist"] >= (1 << 24):
        out |= call_routes(np.diff(r["block"].graph_ptr)[:nx], "real", L, "fw")
    if fit["n_columns"] * 2 > DICT_CAP0:
        out.add("dict_regrow")
    if fit["n_pairs"] > ft_cap0(int(r["block"].graph_ptr[nx]), len(r["label_sets"])):
        out.add("ft_regrow")
    if c["kind"] == "real" and fit["n_lengths"] > c.get("dkey0", DKEY_CAP0):
        out.add("dkey_regrow")
    return out
