// GraphletSampling, sampled route (graphlet_sampling.py, `sampling` a dict; Shervashidze et al. 2009).
//
// Every sample of m <= 6 vertices (drawn on the host: gs_draw) is the reference's undirected bliss graph: a pair
// (i, j) is an edge when the 0/1 adjacency has (i, j) or (j, i), a diagonal entry is a self-loop.  Its pattern has one
// bit per vertex pair (i < j, row-major over the upper triangle) and then one bit per loop, T(m) = m (m - 1) / 2 + m
// bits; the patterns of all sizes share one code space, size m starting at GS_BASE[m].  The class of a pattern is the
// least pattern over the m! relabelings (gs_canon, a table over the whole code space built once per handle), so two
// samples are in one class exactly when the reference's `isomorphic` puts them in one bin.
//
// Counts (graph_bins / local_values of parse_input): the (graph, class) table counts the samples n_ib; the first graph
// in input order that has class b keeps n_ib, every other graph gets n_ib + 1.  In a transform the classes of the
// fitted graphs give every new graph n_ib + 1, and a class only the new graphs have counts from its first new graph.
#pragma once
#include "common.cuh"
#include "wl.cuh"

namespace gk {

constexpr int GS_KMAX = 6;
constexpr unsigned GS_NONE = 0xFFFFFFFFu;
// first code of size m (m = 0 .. 6) and the end of the code space: GS_BASE[m + 1] = GS_BASE[m] + 2^T(m)
__host__ __device__ inline long long gs_base(int m) {
  long long b = 0;
  for (int j = 0; j < m; ++j) b += 1LL << (j * (j - 1) / 2 + j);
  return b;
}

__device__ __forceinline__ int gs_pair_bit(int a, int b, int m) {  // a < b
  return a * (2 * m - a - 1) / 2 + (b - a - 1);
}

// ---- canonical table: canon[c] = GS_BASE[m] + the least pattern of c's relabelings (one thread per code)
__global__ void __launch_bounds__(256) gs_canon(long long n_codes, unsigned* __restrict__ canon) {
  const long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_codes) return;
  int m = 0;
  while (m < GS_KMAX && c >= gs_base(m + 1)) ++m;
  const long long base = gs_base(m);
  const unsigned pat = (unsigned)(c - base);
  const int P = m * (m - 1) / 2;
  int fact = 1;
  for (int j = 2; j <= m; ++j) fact *= j;
  unsigned best = pat;
  for (int t = 0; t < fact; ++t) {
    // permutation number t (factorial number system), 3 bits per image
    unsigned perm = 0, avail = (1u << m) - 1;
    int rest = t, f = fact;
    for (int i = 0; i < m; ++i) {
      f /= (m - i);
      int q = rest / f;
      rest -= q * f;
      unsigned a = avail;
      for (; q > 0; --q) a &= a - 1;
      const int img = __ffs(a) - 1;
      avail &= ~(1u << img);
      perm |= (unsigned)img << (3 * i);
    }
    unsigned out = 0;
    for (int a = 0; a < m; ++a) {
      const int pa = (perm >> (3 * a)) & 7;
      if ((pat >> (P + a)) & 1u) out |= 1u << (P + pa);
      for (int b = a + 1; b < m; ++b) {
        if (!((pat >> gs_pair_bit(a, b, m)) & 1u)) continue;
        const int pb = (perm >> (3 * b)) & 7;
        out |= 1u << (pa < pb ? gs_pair_bit(pa, pb, m) : gs_pair_bit(pb, pa, m));
      }
    }
    best = out < best ? out : best;
  }
  canon[c] = (unsigned)(base + best);
}

// is v an out-neighbour of u (packed CSR, rows ascending)
__device__ __forceinline__ bool gs_has(const int* __restrict__ row_ptr, const int* __restrict__ col_idx, int u, int v) {
  int lo = row_ptr[u], hi = row_ptr[u + 1];
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    const int c = col_idx[mid];
    if (c == v) return true;
    if (c < v) lo = mid + 1; else hi = mid;
  }
  return false;
}

// (graph, class) += c in an open-addressing table of `mask + 1` slots, keys graph << 32 | class
__device__ __forceinline__ void gs_table_add(unsigned long long key, unsigned c, unsigned long long* __restrict__ keys,
                                             unsigned* __restrict__ cnt, unsigned mask) {
  unsigned s = (unsigned)mix64(key) & mask;
  for (;;) {
    unsigned long long cur = keys[s];
    if (cur == EMPTY64) {
      cur = atomicCAS(&keys[s], EMPTY64, key);
      if (cur == EMPTY64) cur = key;
    }
    if (cur == key) { atomicAdd(&cnt[s], c); return; }
    s = (s + 1) & mask;
  }
}

struct GsSampleParams {
  int g0, g1;                  // graphs whose samples are given
  const long long* samp_off;   // [g1 - g0 + 1] first sample of each graph
  const long long* idx_off;    // [g1 - g0 + 1] first index of each graph
  const unsigned char* size;   // [samples] vertices of each sample
  const int* idx;              // drawn vertex indexes, local to their graph
  const int *graph_ptr, *row_ptr, *col_idx;
  const unsigned* canon;
  int n_fit;
  unsigned long long* keys;
  unsigned* cnt;
  unsigned mask;
  unsigned *first_fit, *first_new;  // [n_codes] least graph with the class among the fitted / the new graphs
  unsigned* err;
};

// One warp per graph, 32 samples at a time: a lane's indexes start at the warp's prefix sum of the sizes.
__global__ void __launch_bounds__(256) gs_classify(GsSampleParams p) {
  const int lane = threadIdx.x & 31;
  const int n_graphs = p.g1 - p.g0;
  for (int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < n_graphs; w += (gridDim.x * blockDim.x) >> 5) {
    const int g = p.g0 + w;
    const int v0 = p.graph_ptr[g], n = p.graph_ptr[g + 1] - v0;
    const long long s_end = p.samp_off[w + 1];
    long long io = p.idx_off[w];
    for (long long s0 = p.samp_off[w]; s0 < s_end; s0 += 32) {
      const long long s = s0 + lane;
      const int m = s < s_end ? p.size[s] : 0;
      int pre = m;
      for (int d = 1; d < 32; d <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, pre, d);
        if (lane >= d) pre += t;
      }
      const long long my = io + pre - m;
      io += __shfl_sync(0xffffffffu, pre, 31);
      if (s >= s_end) continue;
      if (m > GS_KMAX) { atomicOr(p.err, 1u); continue; }
      unsigned v[GS_KMAX];
      bool bad = false;
#pragma unroll
      for (int i = 0; i < GS_KMAX; ++i) {
        const int x = i < m ? p.idx[my + i] : 0;
        bad |= x < 0 || x >= n;
        v[i] = (unsigned)(v0 + x);
      }
      if (bad) { atomicOr(p.err, 2u); continue; }
      const int P = m * (m - 1) / 2;
      unsigned pat = 0;
#pragma unroll
      for (int a = 0; a < GS_KMAX; ++a) {
        if (a >= m) break;
        if (gs_has(p.row_ptr, p.col_idx, v[a], v[a])) pat |= 1u << (P + a);
#pragma unroll
        for (int b = a + 1; b < GS_KMAX; ++b) {
          if (b >= m) break;
          if (gs_has(p.row_ptr, p.col_idx, v[a], v[b]) || gs_has(p.row_ptr, p.col_idx, v[b], v[a]))
            pat |= 1u << gs_pair_bit(a, b, m);
        }
      }
      const unsigned code = p.canon[gs_base(m) + pat];
      gs_table_add(((unsigned long long)(unsigned)g << 32) | code, 1u, p.keys, p.cnt, p.mask);
      atomicMin(g < p.n_fit ? &p.first_fit[code] : &p.first_new[code], (unsigned)g);
    }
  }
}

// the rows (graph, class, samples) of an earlier run: graphs kept from a fit without redrawing them
__global__ void __launch_bounds__(256) gs_prior(long long n, const long long* __restrict__ prior, int n_fit,
                                                unsigned long long* keys, unsigned* cnt, unsigned mask,
                                                unsigned* first_fit, unsigned* first_new) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned g = (unsigned)prior[3 * i], code = (unsigned)prior[3 * i + 1];
  gs_table_add(((unsigned long long)g << 32) | code, (unsigned)prior[3 * i + 2], keys, cnt, mask);
  atomicMin((int)g < n_fit ? &first_fit[code] : &first_new[code], g);
}

// dense column of every class some graph has
__global__ void __launch_bounds__(256) gs_number(long long n_codes, const unsigned* __restrict__ first_fit,
                                                 const unsigned* __restrict__ first_new, unsigned* __restrict__ colid,
                                                 unsigned long long* n_cols) {
  const long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_codes) return;
  colid[c] = (first_fit[c] != GS_NONE || first_new[c] != GS_NONE) ? (unsigned)atomicAdd(n_cols, 1ULL) : GS_NONE;
}

// The table in the integer Gram's layout: keys graph << 32 | column, counts with the "+1" rule; the sample counts and
// class codes stay in raw / code.  Rewritten in place, so the table is read linearly from here on, never probed.
__global__ void __launch_bounds__(256) gs_finish(size_t cap, int n_fit, const unsigned* __restrict__ first_fit,
                                                 const unsigned* __restrict__ first_new,
                                                 const unsigned* __restrict__ colid, unsigned long long* __restrict__ keys,
                                                 unsigned* __restrict__ cnt, unsigned* __restrict__ raw,
                                                 unsigned* __restrict__ code_of) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < cap; i += (size_t)gridDim.x * blockDim.x) {
    const unsigned long long k = keys[i];
    if (k == EMPTY64) continue;
    const unsigned g = (unsigned)(k >> 32), code = (unsigned)k;
    const unsigned n = cnt[i];
    unsigned plus;
    if ((int)g < n_fit) plus = first_fit[code] != g;
    else plus = first_fit[code] != GS_NONE ? 1u : (first_new[code] != g);
    raw[i] = n;
    code_of[i] = code;
    cnt[i] = n + plus;
    keys[i] = ((unsigned long long)g << 32) | colid[code];
  }
}

}  // namespace gk
