"""Which feature block the handle holds.  A feature pass refused by its argument checks leaves the previous block as it
was: the next Gram is bit-identical and the family's read-back still answers.  Another family's pass on the same packed
block retires the first family's read-back: it refuses with GK_ERR_STATE instead of returning data of a block the handle
no longer holds."""
import numpy as np
import pytest

from grakel_b200 import _lib
from grakel_b200.kernels import NeighborhoodSubgraphPairwiseDistance

pytestmark = pytest.mark.gpu

KV_DIRAC_KE_NONE = _lib.GK_SM_KV_DIRAC | _lib.GK_SM_KE_NONE
KV_NONE_KE_NONE = _lib.GK_SM_KV_NONE | _lib.GK_SM_KE_NONE


class Block:
    """Four small connected undirected graphs, labels 0 .. 2 and two attributes per vertex, as a packed CSR block."""

    def __init__(self, sizes=(5, 4, 6, 5), seed=3):
        rng = np.random.default_rng(seed)
        self.sizes, self.N = sizes, len(sizes)
        self.adj, gp = [], [0]
        for n in sizes:
            A = np.zeros((n, n), dtype=bool)
            for v in range(1, n):  # a random spanning tree, then a few more edges
                u = int(rng.integers(v))
                A[u, v] = A[v, u] = True
            for _ in range(n // 2):
                u, v = rng.choice(n, 2, replace=False)
                A[u, v] = A[v, u] = True
            self.adj.append(A)
            gp.append(gp[-1] + n)
        self.graph_ptr, self.V = np.array(gp), gp[-1]
        rp, ci = [0], []
        for g, A in enumerate(self.adj):
            for u in range(A.shape[0]):
                ci += [gp[g] + int(v) for v in np.flatnonzero(A[u])]
                rp.append(len(ci))
        self.row_ptr, self.col_idx, self.E = np.array(rp), np.array(ci, dtype=np.int32), len(ci)
        self.deg = np.diff(self.row_ptr)
        self.labels = rng.integers(0, 3, self.V).astype(np.int32)
        self.attrs = rng.random((self.V, 2))
        self.U = rng.random((1, self.V, 2)) * 0.99  # PyramidMatch embeddings in [0, 1)
        self.pk_u = rng.random((2, 3))
        self.rng = rng

    def pack(self, eng):
        eng.pack(self.graph_ptr, self.row_ptr, self.col_idx, self.labels, None, self.attrs)

    def nspd(self):
        """The block as NeighborhoodSubgraphPairwiseDistance packs it: (graph_ptr, row_ptr, col_idx, labels, edge
        labels, vertex hashes, tokens)."""
        graphs = []
        for g, A in enumerate(self.adj):
            n = A.shape[0]
            edges = [(u, int(v)) for u in range(n) for v in np.flatnonzero(A[u])]
            vl = [str(int(x)) for x in self.labels[self.graph_ptr[g]:self.graph_ptr[g + 1]]]
            graphs.append((n, edges, vl, ["e"] * len(edges)))
        return NeighborhoodSubgraphPairwiseDistance(r=1, d=2)._pack(graphs)


def _rw(eng, b, route=_lib.GK_RW_CG):
    vals = np.ones(b.E)  # symmetric graphs: the transposed CSR is the CSR
    eng.rw_features(route, _lib.GK_RW_INV, 0.01, values=vals, t_row_ptr=b.row_ptr, t_col_idx=b.col_idx, t_values=vals)


def _pk(eng, b, t_max=2):
    eng.pk_features(t_max, 0.5, b.pk_u[:max(t_max, 1)], np.array([0.1, 0.2])[:max(t_max, 1)], 3, 3, b.N,
                    np.repeat(1.0 / b.deg, b.deg))


def _gs(eng, b, k=3):
    sizes = np.full(2 * b.N, 3, dtype=np.uint8)  # two samples of three vertices per graph
    idx = np.tile(np.array([0, 1, 2, 1, 2, 3], dtype=np.int32), b.N)
    eng.gs_features(k, b.N, 0, np.arange(0, 2 * b.N + 1, 2), sizes, idx)


def _nspd(eng, b, r=1):
    _, _, _, _, el, sh, tokens = b.nspd()
    eng.nspd_features(r, 2, sh, el, tokens)


def _pack_nspd(eng, b):
    gp, rp, ci, lab, _, _, _ = b.nspd()
    eng.pack(gp, rp, ci, lab, None, None)


# family: (feature pass, the same pass refused by an argument check, read-back[, pack])
FAMILIES = {
    "wl": (lambda e, b: e.wl_features(2), lambda e, b: e.wl_features(-1), lambda e, b: e.wl_labels(2, b.V)),
    "sp": (lambda e, b: e.sp_features(keep_dist=True), lambda e, b: e.wl_sp_features(-1, keep_dist=True),
           lambda e, b: e.sp_distances(1, b.sizes[1])),
    "gh": (lambda e, b: e.gh_features(_lib.GK_GH_LINEAR), lambda e, b: e.gh_features(7),
           lambda e, b: e.gh_node_maps(2, b.sizes[2])),
    "nh": (lambda e, b: e.nh_features(2, _lib.GK_NH_SIMPLE, 8, [5, 9, 17]),
           lambda e, b: e.nh_features(2, _lib.GK_NH_SIMPLE, 0, [5, 9, 17]), lambda e, b: e.nh_labels(1, b.V)),
    "pm": (lambda e, b: e.pm_features(3, 2, b.U, np.full((1, b.N), 2)),
           lambda e, b: e.pm_features(3, 2, b.U, np.full((1, b.N), 3)), lambda e, b: e.pm_cells(0, 2, b.V, 2)),
    "rw": (_rw, lambda e, b: _rw(e, b, route=9), lambda e, b: e.rw_iterations(b.N, b.N)),
    "pk": (_pk, lambda e, b: _pk(e, b, t_max=0), lambda e, b: e.pk_hashes(1, b.V)),
    "sm": (lambda e, b: e.sm_features(3, np.ones(4), flags=KV_DIRAC_KE_NONE),
           lambda e, b: e.sm_features(3, np.ones(4), flags=KV_DIRAC_KE_NONE | _lib.GK_SM_KV_NONE),
           lambda e, b: e.sm_counts(b.N, 1)),
    "sm_wl": (lambda e, b: e.sm_wl_features(3, 1, None, np.ones(4), flags=KV_NONE_KE_NONE),
              lambda e, b: e.sm_wl_features(3, 0, None, np.ones(4), flags=KV_NONE_KE_NONE),
              lambda e, b: e.sm_wl_counts(b.N, 1)),
    "nspd": (_nspd, lambda e, b: _nspd(e, b, r=-1), lambda e, b: e.nspd_hashes(1, b.V), _pack_nspd),
    "odd": (lambda e, b: e.odd_features(2, b.labels), lambda e, b: e.odd_features(0, b.labels),
            lambda e, b: e.odd_signatures()),
    "gs": (_gs, lambda e, b: _gs(e, b, k=0), lambda e, b: e.gs_counts()),
}


def _same(a, b):
    if isinstance(a, tuple):
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    return np.array_equal(np.asarray(a), np.asarray(b), equal_nan=True)


def _setup(eng, b, name):
    run, refuse, read, *pack = FAMILIES[name]
    if pack:
        pack[0](eng, b)
    else:
        b.pack(eng)
    run(eng, b)
    return refuse, read


@pytest.mark.parametrize("name", list(FAMILIES))
def test_refused_call_keeps_the_block(name):
    b = Block()
    with _lib.engine() as eng:
        refuse, read = _setup(eng, b, name)
        K, xd, _ = eng.gram(b.N)
        got = read(eng, b)
        with pytest.raises(_lib.GrakelB200Error, match=r"^\[-2\] "):
            refuse(eng, b)
        K2, xd2, _ = eng.gram(b.N)
        assert _same(K2, K) and _same(xd2, xd), f"{name}: the Gram after a refused call differs"
        assert _same(read(eng, b), got), f"{name}: the read-back after a refused call differs"


@pytest.mark.parametrize("name", list(FAMILIES))
def test_another_pass_retires_the_read_back(name):
    b = Block()
    with _lib.engine() as eng:
        _, read = _setup(eng, b, name)
        eng.gram(b.N)  # the random walk read-back reports the iterations of the last Gram
        read(eng, b)
        (FAMILIES["nh" if name == "wl" else "wl"][0])(eng, b)
        with pytest.raises(_lib.GrakelB200Error, match=r"^\[-3\] "):
            read(eng, b)
