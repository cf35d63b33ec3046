// NeighborhoodSubgraphPairwiseDistance (neighborhood_subgraph_pairwise_distance.py; Costa & De Grave 2010).
//
// Vertices are the indices 0 .. n-1 of a graph's symbols in sorted order (the reference's adjacency round trip), the
// packed CSR lists every vertex's out-neighbours in ascending order and each graph's edges are numbered in CSR order,
// which is the reference's sorted((i, j)) order.
//
// Levels.  graph.py's produce_neighborhoods grows N[l + 1][i] as the union of N[l][w] over w in N[l][i], so ball l
// has BFS radius R(l) = 2^(l - 1) (l >= 1) and a pair at BFS distance t > 0 is at level 1 + ceil(log2 t).
// nspd_bfs stores that level (255: beyond level max(r, d)) in a u8 matrix per graph.
//
// Hashes.  One thread per vertex v (a workspace slot each, reused grid-stride) runs rho = r .. 0: the sub-edge set
// of (v, rho) as CPython 3.12 builds it (set comprehensions over sorted(edges) and then over the previous set, with
// the table's probing and resizes emulated on the edge ids), every member's label as a sorted list of token ranks,
// and the APHash of the encoding streamed from those lists without materialising it.
#pragma once
#include "common.cuh"

namespace gk {

constexpr unsigned NSPD_FAR = 255u;
constexpr unsigned NSPD_EMPTY = 0xFFFFFFFFu;

// ---- CPython 3.12 tuple hash (xxHash lanes) of a pair of element hashes
__host__ __device__ inline unsigned long long nspd_tuple_hash(long long a, long long b) {
  const unsigned long long P1 = 11400714785074694791ULL, P2 = 14029467366897019727ULL, P5 = 2870177450012600261ULL;
  unsigned long long acc = P5;
  acc += (unsigned long long)a * P2;
  acc = (acc << 31) | (acc >> 33);
  acc *= P1;
  acc += (unsigned long long)b * P2;
  acc = (acc << 31) | (acc >> 33);
  acc *= P1;
  acc += 2ULL ^ (P5 ^ 3527539ULL);
  if (acc == ~0ULL) return 1546275796ULL;
  return acc;
}

// ---- CPython 3.12 set of distinct items (set_add_entry, set_table_resize, set_insert_clean).  Items are never
// equal, so only slot occupancy matters; a slot holds the item id, NSPD_EMPTY when free.  Two buffers of `cap`
// slots each (cap >= the largest table) alternate on resize.
struct NspdSet {
  unsigned* buf[2];
  int cur;
  unsigned long long mask, fill;
};

__host__ __device__ inline void nspd_set_clear(NspdSet& s) {
  s.cur = 0;
  s.mask = 7;
  s.fill = 0;
  for (int k = 0; k < 8; ++k) s.buf[0][k] = NSPD_EMPTY;
}

__host__ __device__ inline void nspd_insert_clean(unsigned* tab, unsigned long long mask, unsigned id,
                                                  unsigned long long hash) {
  unsigned long long perturb = hash, i = hash & mask;
  for (;;) {
    if (tab[i] == NSPD_EMPTY) { tab[i] = id; return; }
    if (i + 9 <= mask) {
      for (int j = 1; j <= 9; ++j)
        if (tab[i + j] == NSPD_EMPTY) { tab[i + j] = id; return; }
    }
    perturb >>= 5;
    i = (i * 5 + 1 + perturb) & mask;
  }
}

// hash_of(id) recomputes an item's hash (resizes reinsert every member)
template <class HashOf>
__host__ __device__ inline void nspd_set_add(NspdSet& s, unsigned id, unsigned long long hash, const HashOf& hash_of) {
  unsigned* tab = s.buf[s.cur];
  unsigned long long mask = s.mask, perturb = hash, i = hash & mask;
  for (;;) {
    const int probes = (i + 9 <= mask) ? 9 : 0;
    for (int p = 0; p <= probes; ++p)
      if (tab[i + p] == NSPD_EMPTY) {
        tab[i + p] = id;
        goto inserted;
      }
    perturb >>= 5;
    i = (i * 5 + 1 + perturb) & mask;
  }
inserted:
  s.fill++;
  if (s.fill * 5 < mask * 3) return;
  {
    const unsigned long long used = s.fill, minused = used > 50000 ? used * 2 : used * 4;
    unsigned long long newsize = 8;
    while (newsize <= minused) newsize <<= 1;
    unsigned* nt = s.buf[s.cur ^ 1];
    for (unsigned long long k = 0; k < newsize; ++k) nt[k] = NSPD_EMPTY;
    for (unsigned long long k = 0; k <= mask; ++k)
      if (tab[k] != NSPD_EMPTY) nspd_insert_clean(nt, newsize - 1, tab[k], hash_of(tab[k]));
    s.cur ^= 1;
    s.mask = newsize - 1;
  }
}

// slots a set of n items can reach: the smallest power of two above 4 n, at least 16
__host__ __device__ inline unsigned long long nspd_set_cap(long long n) {
  unsigned long long c = 16;
  while (c <= 4ULL * (unsigned long long)(n > 0 ? n : 0)) c <<= 1;
  return c;
}

// ---- APHash (Arash Partow) over the first `limit` bytes of a stream, bytes read as signed char
struct NspdHash {
  unsigned h;
  long long i, limit;
  __host__ __device__ inline void byte(unsigned char b) {
    if (i >= limit) return;
    const unsigned c = (unsigned)(int)(signed char)b;
    if ((i & 1) == 0) h ^= ((h << 7) ^ c * (h >> 3));
    else h ^= ~((h << 11) + (c ^ (h >> 5)));
    ++i;
  }
};

struct NspdParams {
  int N, r, d, n_labels;
  const int* graph_ptr;   // [N + 1]
  const int* row_ptr;     // [V + 1]
  const int* col_idx;     // [E] global vertex ids, ascending per row
  const int* labels;      // [V] vertex label ids
  const int* edge_label;  // [E] edge label ids
  const long long* sym_hash;      // [V] hash() of every vertex symbol
  const unsigned char* lvl;       // level matrices, graph g at lvl_off[g], n_g x n_g
  const long long* lvl_off;       // [N + 1]
  const int* tok_rank;            // [(d + 1) * n_labels] rank of str(delta) + "," + str(label) in Python's string order
  const long long* rank_off;      // [n_ranks + 1] UTF-8 bytes of every rank
  const unsigned char* rank_bytes;
  const int* rank_cp;             // code points of every rank
  const long long* el_off;        // [n_elabels + 1] UTF-8 bytes of str(edge label)
  const unsigned char* el_bytes;
  const int* el_cp;
  const unsigned char* selfloop;  // [V]
  unsigned* H;                    // [(r + 1) * V] out
  // per-slot workspace
  unsigned* ws;
  long long slot_words, set_cap, max_e, max_n;
  long long ball;                 // largest ball listed, the root twice included: max_n + 1, 1 when r = 0
  int n_slots;
};

__host__ __device__ inline int nspd_graph_of(const int* gp, int N, int v) {
  int lo = 0, hi = N;  // largest g with gp[g] <= v
  while (hi - lo > 1) {
    const int m = (lo + hi) >> 1;
    if (gp[m] <= v) lo = m; else hi = m;
  }
  return lo;
}

// Dist_pair[(i, j)] of the reference (local ids), -1 when the pair is absent
__host__ __device__ inline int nspd_dist(const NspdParams& p, const unsigned char* L, int n, int g0, int i, int j) {
  if (i == j) return (p.r > 0 && p.d >= 1 && p.selfloop[g0 + i]) ? 1 : 0;
  if (p.r == 0) return -1;
  const unsigned l = L[(long long)i * n + j];
  return l <= (unsigned)p.d ? (int)l : -1;
}

// Words of one hashing slot: two set tables, two edge orders, the ball and its label offsets / lengths, the position
// of every vertex and up to B^2 token ranks (B = the largest ball).  Sized by the largest graph of the call, so one
// large graph at r > 0 shrinks the number of slots every graph shares; at r = 0 every ball is its root (B = 1).
__host__ __device__ inline long long nspd_slot_words(long long set_cap, long long max_e, long long max_n, long long B) {
  return 2 * set_cap + 2 * max_e + 3 * (B + 1) + max_n + B * B;
}

// Hashes H[rho][v] for rho = r .. 0 of one vertex, with workspace `w` (nspd_slot_words words)
__host__ __device__ inline void nspd_vertex(const NspdParams& p, int v, unsigned* w) {
  const int g = nspd_graph_of(p.graph_ptr, p.N, v);
  const int g0 = p.graph_ptr[g], n = p.graph_ptr[g + 1] - g0, lv = v - g0;
  const int e0 = p.row_ptr[g0];
  const unsigned char* L = p.lvl + p.lvl_off[g];
  const long long B = p.ball;
  NspdSet set;
  set.buf[0] = w;
  set.buf[1] = w + p.set_cap;
  unsigned* ord[2] = {w + 2 * p.set_cap, w + 2 * p.set_cap + p.max_e};
  unsigned* sub = ord[1] + p.max_e;  // [B + 1]
  unsigned* lv_off = sub + (B + 1);  // [B + 1]
  unsigned* lv_len = lv_off + (B + 1);
  unsigned* pos_of = lv_len + (B + 1);  // [max_n] local vertex -> position in sub
  unsigned* ranks = pos_of + p.max_n;   // [B * B]
  const long long* sh = p.sym_hash + g0;
  auto edge_hash = [&](unsigned e) {
    const int a = nspd_graph_of(p.row_ptr, p.graph_ptr[p.N], e0 + (int)e) - g0;  // source of edge e (local)
    return nspd_tuple_hash(sh[a], sh[p.col_idx[e0 + e] - g0]);
  };
  int n_prev = 0, which = 0;
  for (int rho = p.r; rho >= 0; --rho) {
    // ---- the ball, sorted, with the root twice at rho = 1 when it has a self-loop
    int m = 0;
    for (int j = 0; j < n; ++j) {
      const bool in = rho == 0 ? j == lv : L[(long long)lv * n + j] <= (unsigned)rho;
      if (!in) continue;
      pos_of[j] = (unsigned)m;
      sub[m++] = (unsigned)j;
      if (rho == 1 && j == lv && p.selfloop[v]) sub[m++] = (unsigned)j;
    }
    auto in_ball = [&](int j) { return rho == 0 ? j == lv : L[(long long)lv * n + j] <= (unsigned)rho; };
    // ---- the sub-edge set
    nspd_set_clear(set);
    if (rho == p.r) {
      for (int a = 0; a < n; ++a) {
        if (!in_ball(a)) continue;
        for (int k = p.row_ptr[g0 + a]; k < p.row_ptr[g0 + a + 1]; ++k) {
          const int b = p.col_idx[k] - g0;
          if (in_ball(b)) nspd_set_add(set, (unsigned)(k - e0), nspd_tuple_hash(sh[a], sh[b]), edge_hash);
        }
      }
    } else {
      const unsigned* prev = ord[which ^ 1];
      for (int k = 0; k < n_prev; ++k) {
        const unsigned e = prev[k];
        const int a = nspd_graph_of(p.row_ptr, p.graph_ptr[p.N], e0 + (int)e) - g0, b = p.col_idx[e0 + e] - g0;
        if (in_ball(a) && in_ball(b)) nspd_set_add(set, e, nspd_tuple_hash(sh[a], sh[b]), edge_hash);
      }
    }
    unsigned* out = ord[which];
    int n_out = 0;
    for (unsigned long long k = 0; k <= set.mask; ++k)
      if (set.buf[set.cur][k] != NSPD_EMPTY) out[n_out++] = set.buf[set.cur][k];
    // ---- vertex labels: sorted token ranks of every member (duplicates included)
    unsigned off = 0;
    for (int a = 0; a < m; ++a) {
      const int i = (int)sub[a];
      lv_off[a] = off;
      unsigned* R = ranks + off;
      int c = 0;
      for (int b = 0; b < m; ++b) {
        const int j = (int)sub[b];
        const int dd = nspd_dist(p, L, n, g0, i, j);
        if (dd < 0) continue;
        const unsigned t = (unsigned)p.tok_rank[(long long)dd * p.n_labels + p.labels[g0 + j]];
        int q = c++;  // insertion sort: lists are ball-sized
        while (q > 0 && R[q - 1] > t) { R[q] = R[q - 1]; --q; }
        R[q] = t;
      }
      lv_len[a] = (unsigned)c;
      off += (unsigned)c;
    }
    // ---- encoding: two passes over the same stream, code points first (APHash's length), then the bytes
    NspdHash hs;
    hs.h = 0xAAAAAAAAu;
    for (int pass = 0; pass < 2; ++pass) {
      long long cp = 0;
      hs.i = 0;
      auto sym = [&](unsigned char ch) { if (pass) hs.byte(ch); else ++cp; };
      auto label = [&](int a) {
        for (unsigned t = 0; t < lv_len[a]; ++t) {
          if (t) sym('|');
          const unsigned rk = ranks[lv_off[a] + t];
          if (pass) {
            for (long long b = p.rank_off[rk]; b < p.rank_off[rk + 1]; ++b) hs.byte(p.rank_bytes[b]);
          } else {
            cp += p.rank_cp[rk];
          }
        }
      };
      for (int a = 0; a < m; ++a) {
        label(a);
        sym(a + 1 < m ? '.' : ':');
      }
      for (int k = 0; k < n_out; ++k) {
        const unsigned e = out[k];
        const int i = nspd_graph_of(p.row_ptr, p.graph_ptr[p.N], e0 + (int)e) - g0, j = p.col_idx[e0 + e] - g0;
        label((int)pos_of[i]);
        sym(',');
        label((int)pos_of[j]);
        sym(',');
        const int el = p.edge_label[e0 + e];
        if (pass) {
          for (long long b = p.el_off[el]; b < p.el_off[el + 1]; ++b) hs.byte(p.el_bytes[b]);
        } else {
          cp += p.el_cp[el];
        }
        sym('_');
      }
      if (!pass) hs.limit = cp;
    }
    p.H[(long long)rho * (p.graph_ptr[p.N]) + v] = hs.h;
    n_prev = n_out;
    which ^= 1;
  }
}

// pos_of of the root is its last position at rho = 1 with a self-loop; both positions carry the same label.

__global__ void nspd_hash(NspdParams p, int V) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= p.n_slots) return;
  unsigned* w = p.ws + (long long)t * p.slot_words;
  for (int v = t; v < V; v += p.n_slots) nspd_vertex(p, v, w);
}

// ---- BFS levels: one thread per source vertex, queue in `q` (same layout as the level matrices, int32)
__global__ void nspd_bfs(int V, int N, const int* __restrict__ graph_ptr, const int* __restrict__ row_ptr,
                         const int* __restrict__ col_idx, const long long* __restrict__ lvl_off, int max_level,
                         unsigned char* lvl, int* q) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= V) return;
  const int g = nspd_graph_of(graph_ptr, N, s);
  const int g0 = graph_ptr[g], n = graph_ptr[g + 1] - g0, ls = s - g0;
  unsigned char* row = lvl + lvl_off[g] + (long long)ls * n;
  int* Q = q + lvl_off[g] + (long long)ls * n;
  for (int j = 0; j < n; ++j) row[j] = (unsigned char)NSPD_FAR;
  row[ls] = 0;
  if (max_level == 0) return;
  // distance t reaches level 1 + ceil(log2 t); the last level's radius is 2^(max_level - 1)
  const long long t_max = max_level >= 62 ? (1LL << 62) : (1LL << (max_level - 1));
  int head = 0, tail = 0;
  Q[tail++] = ls;
  long long t = 0;
  int level_end = tail;
  while (head < tail) {
    if (head == level_end) { ++t; level_end = tail; }
    if (t + 1 > t_max) break;
    const int u = Q[head++];
    // level of the vertices found from u: distance t + 1
    const long long td = t + 1;
    int lv = 1;
    while ((1LL << (lv - 1)) < td) ++lv;
    for (int k = row_ptr[g0 + u]; k < row_ptr[g0 + u + 1]; ++k) {
      const int b = col_idx[k] - g0;
      if (row[b] != (unsigned char)NSPD_FAR) continue;
      row[b] = (unsigned char)lv;
      Q[tail++] = b;
    }
  }
}

// ---- pairs of D[delta]: one CTA per graph.  fill == 0 counts (and sets the graph's delta mask), fill == 1 writes
// the pairs (global ids) at the cursors.
__global__ void nspd_pairs(int N, int r, int d, const int* __restrict__ graph_ptr, const long long* __restrict__ lvl_off,
                           const unsigned char* __restrict__ lvl, const unsigned char* __restrict__ selfloop, int fill,
                           unsigned long long* cnt, unsigned long long* cursor, const unsigned long long* base,
                           unsigned* A, unsigned* Bv, unsigned long long* mask) {
  for (int g = blockIdx.x; g < N; g += gridDim.x) {
    const int g0 = graph_ptr[g], n = graph_ptr[g + 1] - g0;
    const unsigned char* L = lvl + lvl_off[g];
    unsigned long long my_mask = 0;
    for (long long k = threadIdx.x; k < (long long)n * n; k += blockDim.x) {
      const int i = (int)(k / n), j = (int)(k % n);
      int dl[2], nd = 0;
      if (i == j) {
        dl[nd++] = 0;
        if (r > 0 && d >= 1 && selfloop[g0 + i]) dl[nd++] = 1;
      } else if (r > 0 && L[k] <= (unsigned)d) {
        dl[nd++] = L[k];
      }
      for (int t = 0; t < nd; ++t) {
        my_mask |= 1ULL << dl[t];
        if (!fill) {
          atomicAdd(&cnt[dl[t]], 1ULL);
        } else {
          const unsigned long long at = base[dl[t]] + atomicAdd(&cursor[dl[t]], 1ULL);
          A[at] = (unsigned)(g0 + i);
          Bv[at] = (unsigned)(g0 + j);
        }
      }
    }
    if (!fill && my_mask) atomicOr(&mask[g], my_mask);
  }
}

// ---- level (rho, delta) keys: (H[rho, A], H[rho, B]) and the graph of every pair
__global__ void nspd_keys(long long M, const unsigned* __restrict__ A, const unsigned* __restrict__ Bv,
                          const unsigned* __restrict__ Hr, const int* __restrict__ vgraph, unsigned long long* keys,
                          int* egraph) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= M) return;
  keys[e] = ((unsigned long long)Hr[A[e]] << 32) | Hr[Bv[e]];
  egraph[e] = vgraph[A[e]];
}

// ---- statistics of a level's (graph, column) -> count table: graphs per column, self similarities (sum of squared
// counts), largest count and entries (the one partial gram_int folds)
__global__ void nspd_level_stats(size_t cap, const unsigned long long* __restrict__ keys, const unsigned* __restrict__ cnt,
                                 unsigned* colcnt, unsigned long long* diag, unsigned* part) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < cap; i += (size_t)gridDim.x * blockDim.x) {
    const unsigned long long k = keys[i];
    if (k == EMPTY64) continue;
    const unsigned c = cnt[i];
    if (__ldcg(&colcnt[(unsigned)k]) < COL_CAP) atomicAdd(&colcnt[(unsigned)k], 1u);
    atomicAdd(&diag[k >> 32], (unsigned long long)c * c);
    atomicMax(&part[0], c);
    atomicAdd(&part[1], 1u);
  }
}

// ---- fold of one level into K: S += nan_to_num(k / sqrt(d_i * d_j)), the products in int64, every operation one
// correctly rounded IEEE double operation.  In the square case a NaN on the diagonal is 1 (fill_diagonal).
__global__ void nspd_fold(int rows, int cols, const double* __restrict__ C, long long ldc, int row_g0,
                          const unsigned long long* __restrict__ diag, int square, double* out, long long ld) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)rows * cols) return;
  const int i = (int)(t / cols), j = (int)(t % cols);
  const int gi = row_g0 + i;
  const long long k = __double2ll_rn(C[(long long)i * ldc + j]);
  const long long prod = (long long)(diag[gi] * diag[j]);
  double q = __ddiv_rn(__ll2double_rn(k), __dsqrt_rn(__ll2double_rn(prod)));
  if (isnan(q)) q = (square && gi == j) ? 1.0 : 0.0;
  else if (isinf(q)) q = q > 0 ? 1.7976931348623157e308 : -1.7976931348623157e308;
  double* o = out + (long long)i * ld + j;
  *o = __dadd_rn(*o, q);
}

__global__ void nspd_scale(int rows, int cols, double div, double* out, long long ld) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)rows * cols) return;
  double* o = out + (t / cols) * ld + (t % cols);
  *o = __ddiv_rn(*o, div);
}

}  // namespace gk
