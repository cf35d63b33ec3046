"""Inputs for the WL collision tests: "twins" -- pairs of vertices with equal own label and degree whose sorted
neighbour-label multisets differ in exactly one position -- plus helpers that read the oracle's levels.

A twin centre carries label CENTRE and `d` spokes.  depth 1: spoke j ends in a leaf labelled base[j]; the twins split at
level 1.  depth 3: spoke j is a path centre - SPOKE - LINK - leaf(base[j]); the twins share every label up to level 2 and
split at level 3 (the differing leaf is three hops away).  base = 2, 4, .., 2d; the second twin's list changes position
`pos` (first: 1, middle: base[d // 2] + 1, last: 2d + 1) and stays sorted, so the position is the same in the kernels'
sorted order.  Labels stay below 2d + 2 <= 402, CENTRE / SPOKE / LINK are above that."""
import numpy as np

CENTRE, SPOKE, LINK = 1000, 1001, 1002
DEGREES = (1, 2, 5, 6, 7, 8, 9, 16, 17, 32, 33, 64, 200)
POSITIONS = ("first", "middle", "last")


def leaf_labels(d, pos, second):
    base = [2 * (j + 1) for j in range(d)]
    if second:
        j = {"first": 0, "middle": d // 2, "last": d - 1}[pos]
        base[j] = {"first": 1, "middle": base[j] + 1, "last": 2 * d + 1}[pos]
    return base


class _G:
    """Edge dictionary + labels of one graph under construction."""

    def __init__(self):
        self.edges, self.labels = {}, {}

    def vertex(self, label):
        v = len(self.labels)
        self.labels[v] = label
        return v

    def edge(self, u, v):
        self.edges[(u, v)] = 1
        self.edges[(v, u)] = 1

    def twin(self, d, pos, second, depth):
        c = self.vertex(CENTRE)
        for lab in leaf_labels(d, pos, second):
            if depth == 1:
                self.edge(c, self.vertex(lab))
            else:
                s, k, t = self.vertex(SPOKE), self.vertex(LINK), self.vertex(lab)
                self.edge(c, s)
                self.edge(s, k)
                self.edge(k, t)
        return self

    def element(self):
        return [self.edges, self.labels]


def twin_pairs(d, pos, depth=1):
    """The three placements of one twin pair, as lists of graphs:
    both centres in one graph; in two adjacent graphs (one tile of the fused kernel when they are small);
    and (first, last) to be put at the two ends of the block (different tiles and CTAs)."""
    same = _G().twin(d, pos, False, depth).twin(d, pos, True, depth).element()
    adj = [_G().twin(d, pos, False, depth).element(), _G().twin(d, pos, True, depth).element()]
    far = (_G().twin(d, pos, False, depth).element(), _G().twin(d, pos, True, depth).element())
    return same, adj, far


def filler(n_copies, seed=5):
    """Copies of one random graph whose vertex i is labelled 2000 + i: vertex i of every copy has the same signature at
    every level, so the filler adds vertices (a non-trivial tile partition) but no class that splits."""
    from oracle.gk_oracle import gen
    g, lab = gen(1, 20, seed)[0]
    return [[dict(g), {v: 2000 + v for v in lab}] for _ in range(n_copies)]


def block(degrees=DEGREES, positions=POSITIONS, depth3=(), background=()):
    """Every (degree, position) twin pair in its three placements, depth-3 twins for the degrees in `depth3`, and the
    background graphs in the middle."""
    head, mid, tail = [], [], []
    for d in degrees:
        for pos in positions:
            for depth in (1, 3) if d in depth3 else (1,):
                same, adj, (a, b) = twin_pairs(d, pos, depth)
                head.append(a)
                mid += [same] + adj
                tail.append(b)
    return head + mid + list(background) + tail[::-1]


# ---------------------------------------------------------------- reading the oracle
def degrees_of(X):
    """Out-degree of every vertex, graph by graph in sorted vertex order (the packed order of a labels dictionary)."""
    out = []
    for g, lab in X:
        deg = {v: 0 for v in lab}
        for (u, _v) in g:
            deg[u] = deg.get(u, 0) + 1
        out += [deg[v] for v in sorted(lab)]
    return np.asarray(out, dtype=np.int64)


def first_split_level(parts, deg, from_level):
    """First level lv >= from_level at which the partition splits a (level lv-1 label, degree) group -- the first level at
    which a key of own label and degree alone must collide -- or None."""
    for lv in range(max(from_level, 1), len(parts)):
        key = parts[lv - 1] * (int(deg.max()) + 1) + deg
        _, inv = np.unique(key, return_inverse=True)
        # a group splits iff it holds more than one class of level lv
        pairs = np.unique(np.stack([inv.ravel(), parts[lv]], axis=1), axis=0)
        if len(pairs) > inv.max() + 1:
            return lv
    return None


def group_width(deg):
    """The multi-kernel route's signature kernel choice (gk_pack_csr): cost V lanes + 32 per vertex above 8 for the
    thread-per-vertex kernel, 16 V (32 V) lanes + 32 per vertex above 16 (32) for the 16 (32)-lane kernel; the vertices
    above the chosen width go to the warp-per-vertex kernel.  Ties keep the narrower kernel."""
    V = len(deg)
    above = {w: int((deg > w).sum()) for w in (8, 16, 32)}
    cost = {8: V + 32 * above[8], 16: 16 * V + 32 * above[16], 32: 32 * V + 32 * above[32]}
    best = 8
    for w in (16, 32):
        if cost[w] < cost[best]:
            best = w
    return best, above[best]


def degree_mix(width, n_graphs=40, seed=0):
    """Random graphs whose degrees make the multi-kernel route pick `width`, each with one hub above the width."""
    rs = np.random.RandomState(seed + width)
    n, p = {8: (20, 0.2), 16: (40, 0.3), 32: (64, 0.35)}[width]
    X = []
    for _ in range(n_graphs):
        A = np.triu(rs.rand(n, n) < p, 1)
        A = A | A.T
        A[0, 1:] = A[1:, 0] = True  # hub: degree n - 1 > width
        g = {(int(u), int(v)): 1 for u, v in zip(*np.nonzero(A))}
        X.append([g, {i: int(rs.randint(3)) for i in range(n)}])
    return X
