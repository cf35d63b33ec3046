"""NumPy restatement of the level-1 signature key of the fused WL relabel kernel (wl_fused2.cuh [A1], degree <= 8) and
of its hash-table placement, for the natural-collision test.

Key: wlf_seq_step over the sorted neighbour labels from (0x243F6A88, 0x85A308D3), then wlf_finish with the first-attempt
seed mix64(0x5851F42D4C957F2D) (wl_fused2.cuh).  Table: the start slot ((key & 0xFFFFFFFF) * 0x9E3779B1 >> 8) & mask and
the tag key >> 33 ([A3]).  Two distinct signatures with equal tag and start slot meet in one slot and only the
verification in [B] can tell them apart.  If the kernel's hash changes, this file must change with it (the GPU test
then sees no collision)."""
import numpy as np

M32 = np.uint64(0xFFFFFFFF)
M64 = (1 << 64) - 1


def mix64(x):
    x &= M64
    x ^= x >> 33
    x = (x * 0xFF51AFD7ED558CCD) & M64
    x ^= x >> 33
    x = (x * 0xC4CEB9FE1A85EC53) & M64
    x ^= x >> 33
    return x


SEED0 = mix64(0x5851F42D4C957F2D)  # attempt 0 of gk_wl_features and the asynchronous pass of gk_wl_gram


def _u32(x):
    return x & M32


def _fmix(h):
    h = h ^ (h >> np.uint64(16))
    h = _u32(h * np.uint64(0x85EBCA6B))
    h = h ^ (h >> np.uint64(13))
    h = _u32(h * np.uint64(0xC2B2AE35))
    return h ^ (h >> np.uint64(16))


def key_level1(own, nbrs, seed=SEED0):
    """Keys of n vertices: own[n] labels, nbrs[n, d] SORTED neighbour labels (d <= 8, equal for all rows)."""
    nbrs = np.asarray(nbrs)
    n, deg = nbrs.shape
    assert deg <= 8
    a = np.full(n, 0x243F6A88, np.uint64)
    c = np.full(n, 0x85A308D3, np.uint64)
    for j in range(deg):  # wlf_seq_step
        x = nbrs[:, j].astype(np.uint64)
        a = _u32((a ^ x) * np.uint64(0x9E3779B1))
        a ^= a >> np.uint64(15)
        c = _u32((c + x) * np.uint64(0x85EBCA77))
        c ^= c >> np.uint64(13)
    o = np.asarray(own).astype(np.uint64)  # wlf_finish
    a = _fmix(a ^ _u32(o * np.uint64(0x9E3779B1)) ^ np.uint64(seed & 0xFFFFFFFF))
    c = _fmix(_u32(c + o * np.uint64(0x7FEB352D) + np.uint64(deg) * np.uint64(0x846CA68B) + np.uint64(seed >> 32)))
    return ((a << np.uint64(32)) | c) >> np.uint64(1)


def start_slot(key, ht_cap):
    return ((key & M32) * np.uint64(0x9E3779B1) >> np.uint64(8)) & np.uint64(ht_cap - 1)


def tag(key):
    return key >> np.uint64(33)


def find_colliding_pair(seed=0, n=4_000_000, n_labels=64, deg=8, ht_cap=1024):
    """Birthday search over random (own label, `deg` sorted neighbour labels) tuples drawn from `n_labels` labels: the
    first pair (in key order) of DISTINCT signatures with equal tag and equal start slot in a table of `ht_cap` slots.
    Returns ((own_a, nbrs_a), (own_b, nbrs_b)) as Python ints / lists, or None."""
    rs = np.random.RandomState(seed)
    own = rs.randint(0, n_labels, n).astype(np.uint8)
    nb = np.sort(rs.randint(0, n_labels, (n, deg)).astype(np.uint8), axis=1)
    k = key_level1(own, nb)
    comb = (tag(k) << np.uint64(int(ht_cap - 1).bit_length())) | start_slot(k, ht_cap)
    order = np.argsort(comb, kind="stable")
    cs = comb[order]
    for h in np.flatnonzero(cs[1:] == cs[:-1]).tolist():
        i, j = int(order[h]), int(order[h + 1])
        if own[i] != own[j] or not np.array_equal(nb[i], nb[j]):
            return (int(own[i]), nb[i].tolist()), (int(own[j]), nb[j].tolist())
    return None
