// Shortest-path kernel features on the device: batched Floyd-Warshall (one CTA per
// graph, distance matrix in shared memory) + labelled path-length histogram.
//
// Replaces Graph.build_shortest_path_matrix / floyd_warshall / dijkstra
// (graph.py:588-687, 1767-1794, 1712-1764) and the pair loop of
// ShortestPath.parse_input (shortest_path.py:468-490) of the reference:
//   for every ordered pair u != v with finite distance, feature (l(u), l(v), d(u,v))
//   (or just d(u,v) when with_labels=False) is counted once.
// Both reference algorithms return exact shortest distances; for integer-valued
// weights those are order-independent integers, which is what this path supports
// (a non-integer distance raises GK_ERR_UNSUPPORTED instead of guessing a key).
#pragma once
#include "common.cuh"
#include "wl.cuh"

namespace gk {

constexpr int SP_LOCAL_SLOTS = 2048;  // per-CTA (key -> count) aggregation table
constexpr int SP_THREADS = 256;
constexpr int SP_DIRECT_MAX_LABELS = 11;  // sp_bfs_hist: direct (ls, lv, level) counters up to this alphabet size

template <typename T> struct DistTraits;
template <> struct DistTraits<unsigned short> {
  static __device__ __forceinline__ unsigned short inf() { return 0x3FFF; }
  static __device__ __forceinline__ unsigned short add(unsigned short a, unsigned short b) {
    unsigned s = (unsigned)a + b;
    return (unsigned short)(s > 0x3FFFu ? 0x3FFFu : s);
  }
  static __device__ __forceinline__ bool finite(unsigned short a) { return a < 0x3FFF; }
  static __device__ __forceinline__ double to_f64(unsigned short a) {
    return a < 0x3FFF ? (double)a : __longlong_as_double(0x7ff0000000000000LL);
  }
};
template <> struct DistTraits<double> {
  static __device__ __forceinline__ double inf() { return __longlong_as_double(0x7ff0000000000000LL); }
  static __device__ __forceinline__ double add(double a, double b) { return a + b; }
  static __device__ __forceinline__ bool finite(double a) { return a < 1.0e300; }
  static __device__ __forceinline__ double to_f64(double a) { return a; }
};

struct SpParams {
  const int* graph_ptr;
  const int* row_ptr;
  const int* col_idx;
  const double* weights;   // NULL = unit
  const int* labels;       // dense ids or NULL (with_labels = False)
  int label_offset;        // added to every label (WL levels share one dictionary: ids are made level-unique)
  const int* glist;        // graphs handled by this launch (NULL = all, blockIdx.x)
  int n_list;
  int n_labels;            // size of the label alphabet (1 when with_labels = False)
  void* gdist;             // global distance scratch (large graphs / keep_dist)
  const long long* goff;   // element offset of graph g inside gdist
  int dist_in_global;      // 1: run FW in gdist instead of shared memory
  double* keep;            // if non-NULL: write fp64 distances of every graph at keep + goff[g]
  unsigned long long* dict_keys;
  unsigned dict_mask;
  unsigned long long* ft_keys;
  unsigned* ft_cnt;
  unsigned ft_mask;
  DevScalars* sc;
  FeatStats st;
};

// one ft_add of `inc` occurrences + its self-similarity / max-count bookkeeping
__device__ __forceinline__ void sp_feature_add(const SpParams& p, int g, int col, unsigned inc) {
  bool is_new;
  const unsigned old = ft_add(p.ft_keys, p.ft_cnt, p.ft_mask, ((unsigned long long)(unsigned)g << 32) | (unsigned)col,
                              inc, p.st, &is_new);
  atomicAdd(&p.st.diag[g], (unsigned long long)inc * (2ULL * old + inc));  // (old+inc)^2 - old^2
  // graph g is owned by this CTA: its partial slots are private to the block (smem-free, L2 atomics
  // on a per-CTA address do not contend across CTAs)
  atomicMax(&p.st.part_max[blockIdx.x], old + inc);
  if (is_new) atomicAdd(&p.st.part_new[blockIdx.x], 1u);
}

// open-addressing insert into a global key table: returns the key's slot; a new key adds 1 to *size.  A table that is
// full -- or has a probe chain longer than SP_TABLE_PROBES, which the host's load limit of one half makes vanishingly
// rare -- sets `ovf_bit` in ft_overflow and returns 0: the host grows that table and repeats the call.  Once the bit
// is set the attempt is void, so later inserts return at once instead of sweeping a full table each.
constexpr unsigned SP_TABLE_PROBES = 4096;
__device__ __forceinline__ int sp_table_slot(unsigned long long* keys, unsigned mask, unsigned long long key,
                                             unsigned* size, DevScalars* sc, unsigned ovf_bit) {
  if (__ldcg(&sc->ft_overflow) & ovf_bit) return 0;
  unsigned slot = (unsigned)(mix64(key) >> 13) & mask;
  const unsigned probes = mask < SP_TABLE_PROBES ? mask + 1 : SP_TABLE_PROBES;
  for (unsigned probe = 0; probe < probes; ++probe) {
    unsigned long long prev = __ldcg(&keys[slot]);
    if (prev == EMPTY64) {
      prev = atomicCAS(&keys[slot], EMPTY64, key);
      if (prev == EMPTY64) { atomicAdd(size, 1u); return (int)slot; }
    }
    if (prev == key) return (int)slot;
    slot = (slot + 1) & mask;
  }
  atomicOr(&sc->ft_overflow, ovf_bit);
  return 0;
}

// global (lu,lv,d) dictionary: the slot index IS the column id
__device__ __forceinline__ int sp_dict_slot(unsigned long long* keys, unsigned mask, unsigned long long key,
                                            DevScalars* sc) {
  return sp_table_slot(keys, mask, key, &sc->sp_dict_size, sc, 2u);
}

// global dictionary of distinct path lengths (real mode, SP-attr): counted apart from the feature columns, and with
// an overflow bit of its own (8) so that only the table that overflowed is grown
__device__ __forceinline__ int sp_dkey_slot(unsigned long long* keys, unsigned mask, unsigned long long key,
                                            DevScalars* sc) {
  return sp_table_slot(keys, mask, key, &sc->sp_dkey_size, sc, 8u);
}

// CTA-local (key -> count) aggregation shared by the SP feature kernels; falls through to
// the global tables when the probe window is full.
__device__ __forceinline__ void sp_local_add(unsigned long long* lkeys, unsigned* lcnt, const SpParams& p, int g,
                                             unsigned long long key) {
  unsigned slot = (unsigned)(mix64(key) >> 29) & (SP_LOCAL_SLOTS - 1);
  for (int probe = 0; probe < 16; ++probe) {
    unsigned long long prev = lkeys[slot];
    if (prev == EMPTY64) prev = atomicCAS(&lkeys[slot], EMPTY64, key);
    if (prev == EMPTY64 || prev == key) { atomicAdd(&lcnt[slot], 1u); return; }
    slot = (slot + 1) & (SP_LOCAL_SLOTS - 1);
  }
  const int col = sp_dict_slot(p.dict_keys, p.dict_mask, key, p.sc);
  sp_feature_add(p, g, col, 1u);
}

// Unit-weight graphs: all-sources BFS on adjacency BITMASKS instead of Floyd-Warshall.
// One CTA per graph, one thread per source vertex; visited / frontier sets are W 64-bit
// words in registers (n <= 64*W).  Every newly reached vertex v at BFS level d is exactly
// one ordered pair (s, v) with shortest distance d (graph.py:1712-1764 computes the same
// distances), so the (l(s), l(v), d) feature is counted on the spot and no n x n distance
// matrix is materialised: O(n (n + m)/64) word operations per graph instead of n^3
// min-plus steps.
template <int W>
__global__ void __launch_bounds__(128)
sp_bfs_hist(SpParams p) {
  extern __shared__ __align__(16) unsigned char sp_smem[];
  const int g = p.glist ? p.glist[blockIdx.x] : blockIdx.x;
  const int v0 = p.graph_ptr[g];
  const int n = p.graph_ptr[g + 1] - v0;
  if (n <= 0) return;
  // Small alphabets (L <= 11): the CTA-local histogram is DIRECT-indexed by (ls, lv, level) --
  // one shared-memory atomicAdd per (source, level, label class) with the class population count,
  // instead of a hashed CAS + add per vertex pair (shared atomics cost ~2 cycles per lane).
  // The direct table needs counters only, so the 16 KB key array is not allocated in that mode
  // (3x more resident CTAs per SM): layout [keys (hashed mode only) | counts | adj | lmask | labels].
  const int L = p.n_labels;
  const bool direct = L <= SP_DIRECT_MAX_LABELS;  // >= 16 levels in the direct table; deeper levels go to the global table
  const int dcap = direct ? SP_LOCAL_SLOTS / (L * L) : 0;  // levels covered by the direct table
  unsigned long long* lkeys = reinterpret_cast<unsigned long long*>(sp_smem);
  unsigned* lcnt = reinterpret_cast<unsigned*>(sp_smem + (direct ? 0 : SP_LOCAL_SLOTS * 8));
  unsigned long long* adj = reinterpret_cast<unsigned long long*>(sp_smem + (direct ? SP_LOCAL_SLOTS * 4 : SP_LOCAL_SLOTS * 12));  // [n][W]
  unsigned long long* lmask = adj + (size_t)n * W;                                                  // [L][W] (direct mode)
  int* lab = reinterpret_cast<int*>(lmask + (direct ? (size_t)L * W : 0));                          // [n]
  const int tid = threadIdx.x;
  for (int i = tid; i < SP_LOCAL_SLOTS; i += blockDim.x) { if (!direct) lkeys[i] = EMPTY64; lcnt[i] = 0; }
  for (int i = tid; i < n * W; i += blockDim.x) adj[i] = 0ULL;
  if (direct) for (int i = tid; i < L * W; i += blockDim.x) lmask[i] = 0ULL;
  for (int i = tid; i < n; i += blockDim.x) lab[i] = p.labels ? p.labels[v0 + i] + p.label_offset : 0;
  __syncthreads();
  const int e0 = p.row_ptr[v0], e1 = p.row_ptr[v0 + n];
  // edge list -> bitmask rows (vertex of edge k found by binary search in row_ptr)
  for (int k = e0 + tid; k < e1; k += blockDim.x) {
    int lo = 0, hi = n;
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (p.row_ptr[v0 + mid] <= k) lo = mid; else hi = mid;
    }
    const int w = p.col_idx[k] - v0;
    if (w != lo) atomicOr(&adj[(size_t)lo * W + (w >> 6)], 1ULL << (w & 63));
  }
  if (direct)
    for (int v = tid; v < n; v += blockDim.x) atomicOr(&lmask[(size_t)lab[v] * W + (v >> 6)], 1ULL << (v & 63));
  __syncthreads();
  double* keep = p.keep ? p.keep + p.goff[g] : nullptr;
  for (int s = tid; s < n; s += blockDim.x) {
    unsigned long long vis[W], fr[W], nx[W];
#pragma unroll
    for (int w = 0; w < W; ++w) { fr[w] = adj[(size_t)s * W + w]; vis[w] = fr[w]; }
#pragma unroll
    for (int w = 0; w < W; ++w)
      if (w == (s >> 6)) vis[w] |= 1ULL << (s & 63);
    if (keep) {
      for (int v = 0; v < n; ++v) keep[(size_t)s * n + v] = __longlong_as_double(0x7ff0000000000000LL);
      keep[(size_t)s * n + s] = 0.0;
    }
    const int lsi = lab[s];
    const unsigned long long ls = (unsigned long long)(unsigned)lsi;
    unsigned level = 1;
    while (true) {
      bool any = false;
#pragma unroll
      for (int w = 0; w < W; ++w) { nx[w] = 0ULL; any |= fr[w] != 0ULL; }
      if (!any) break;
      const bool use_direct = direct && (int)level <= dcap;
      if (use_direct) {  // class population counts of the new frontier
        for (int l = 0; l < L; ++l) {
          int c = 0;
#pragma unroll
          for (int w = 0; w < W; ++w) c += __popcll(fr[w] & lmask[(size_t)l * W + w]);
          if (c) atomicAdd(&lcnt[(lsi * L + l) * dcap + (int)level - 1], (unsigned)c);
        }
      }
#pragma unroll
      for (int w = 0; w < W; ++w) {
        unsigned long long bits = fr[w];
        while (bits) {
          const int b = __ffsll((long long)bits) - 1;
          bits &= bits - 1;
          const int v = (w << 6) + b;
          if (!use_direct) {
            const unsigned long long key = (ls << 44) | ((unsigned long long)(unsigned)lab[v] << 24) | level;
            if (direct) {  // level beyond the direct table: lcnt holds direct counters, bypass the CTA table
              const int col = sp_dict_slot(p.dict_keys, p.dict_mask, key, p.sc);
              sp_feature_add(p, g, col, 1u);
            } else {
              sp_local_add(lkeys, lcnt, p, g, key);
            }
          }
          if (keep) keep[(size_t)s * n + v] = (double)level;
#pragma unroll
          for (int x = 0; x < W; ++x) nx[x] |= adj[(size_t)v * W + x];
        }
      }
#pragma unroll
      for (int w = 0; w < W; ++w) { nx[w] &= ~vis[w]; vis[w] |= nx[w]; fr[w] = nx[w]; }
      ++level;
    }
  }
  __syncthreads();
  for (int i = tid; i < SP_LOCAL_SLOTS; i += blockDim.x) {
    unsigned long long key;
    const unsigned c = lcnt[i];
    if (direct) {  // slot i = (ls * L + lv) * dcap + (level - 1)
      if (!c || i >= L * L * dcap) continue;
      const int pair = i / dcap, lev = i - pair * dcap + 1;
      key = ((unsigned long long)(pair / L) << 44) | ((unsigned long long)(pair % L) << 24) | (unsigned long long)lev;
    } else {
      key = lkeys[i];
      if (key == EMPTY64) continue;
    }
    const int col = sp_dict_slot(p.dict_keys, p.dict_mask, key, p.sc);
    sp_feature_add(p, g, col, c);
  }
}

template <typename T>
__global__ void __launch_bounds__(SP_THREADS)
sp_apsp_hist(SpParams p) {
  using DT = DistTraits<T>;
  extern __shared__ __align__(16) unsigned char sp_smem[];
  const int g = p.glist ? p.glist[blockIdx.x] : blockIdx.x;
  const int v0 = p.graph_ptr[g];
  const int n = p.graph_ptr[g + 1] - v0;
  if (n <= 0) return;

  // smem carve-up: [local keys | local counts | labels? no: labels read from global | dist]
  unsigned long long* lkeys = reinterpret_cast<unsigned long long*>(sp_smem);
  unsigned* lcnt = reinterpret_cast<unsigned*>(sp_smem + SP_LOCAL_SLOTS * 8);
  T* dist = p.dist_in_global ? reinterpret_cast<T*>(p.gdist) + p.goff[g]
                             : reinterpret_cast<T*>(sp_smem + SP_LOCAL_SLOTS * 12);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  constexpr int NW = SP_THREADS / 32;

  for (int i = tid; i < SP_LOCAL_SLOTS; i += SP_THREADS) { lkeys[i] = EMPTY64; lcnt[i] = 0; }
  const long long nn = (long long)n * n;
  for (long long i = tid; i < nn; i += SP_THREADS) dist[i] = DT::inf();
  __syncthreads();
  // adjacency -> initial distances (graph.py:1785-1787: 0 entries are "no edge", diagonal 0)
  for (int u = warp; u < n; u += NW) {
    const int b = p.row_ptr[v0 + u], e = p.row_ptr[v0 + u + 1];
    for (int k = b + lane; k < e; k += 32) {
      const int w = p.col_idx[k] - v0;
      if (w == u) continue;
      if constexpr (sizeof(T) == 2) {
        dist[(long long)u * n + w] = 1;
      } else {
        dist[(long long)u * n + w] = p.weights ? (T)p.weights[k] : (T)1;
      }
    }
    if (lane == 0) dist[(long long)u * n + u] = 0;
  }
  __syncthreads();
  // classic k-ordered relaxation (graph.py:1790-1792); rows whose d[i][k] is infinite
  // cannot improve and are skipped.
  for (int k = 0; k < n; ++k) {
    const T* rk = dist + (long long)k * n;
    for (int i = warp; i < n; i += NW) {
      if (i == k) continue;
      T* ri = dist + (long long)i * n;
      const T dik = ri[k];
      if (!DT::finite(dik)) continue;
      for (int j = lane; j < n; j += 32) {
        const T cand = DT::add(dik, rk[j]);
        if (cand < ri[j]) ri[j] = cand;
      }
    }
    __syncthreads();
  }
  if (p.keep) {
    double* o = p.keep + p.goff[g];
    for (long long i = tid; i < nn; i += SP_THREADS) o[i] = DT::to_f64(dist[i]);
  }
  // labelled path-length histogram (shortest_path.py:470-490)
  for (int u = warp; u < n; u += NW) {
    const unsigned long long lu = p.labels ? (unsigned long long)(unsigned)(p.labels[v0 + u] + p.label_offset) : 0ULL;
    const T* ru = dist + (long long)u * n;
    for (int w = lane; w < n; w += 32) {
      if (w == u) continue;
      const T d = ru[w];
      if (!DT::finite(d)) continue;
      unsigned di;
      if constexpr (sizeof(T) == 2) {
        di = d;
      } else {
        di = (unsigned)d;
        if ((double)di != (double)d || d >= 16777216.0) { atomicOr(&p.sc->sp_nonint, 1u); continue; }
      }
      const unsigned long long lv = p.labels ? (unsigned long long)(unsigned)(p.labels[v0 + w] + p.label_offset) : 0ULL;
      const unsigned long long key = (lu << 44) | (lv << 24) | (unsigned long long)di;
      sp_local_add(lkeys, lcnt, p, g, key);
    }
  }
  __syncthreads();
  for (int i = tid; i < SP_LOCAL_SLOTS; i += SP_THREADS) {
    const unsigned long long key = lkeys[i];
    if (key == EMPTY64) continue;
    const int col = sp_dict_slot(p.dict_keys, p.dict_mask, key, p.sc);
    sp_feature_add(p, g, col, lcnt[i]);
  }
}

}  // namespace gk
