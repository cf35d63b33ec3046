// PyramidMatch (Nikolentzos et al. 2017; pyramid_match.py:18-285) on the device.
//
// The vertex embeddings |U| (eigenvectors of the adjacency matrix) come from the host: they are made by the same
// scipy / numpy calls as the reference, so K equals the reference's bit for bit given the same U.  Level j < L puts
// entry (vertex v, dimension q < n_cols) into cell T = floor(u * 2^j) (T == 2^j clamped to 2^j - 1) of histogram row
// label(v) * d + q (or q without labels).  Every (level, row, cell) is one u64 key (row << j | T); the keys of a level
// are numbered and counted per graph by the NeighborhoodHash column pipeline (neighborhood_hash.cuh, d entries per
// vertex), unary-expanded (wl_oa.cuh), and the exact integer Gram of each level gives the intersections
// I_j(x, y) = sum min(cnt_x, cnt_y).  pm_combine then replays the reference's fp64 combine of the I_j.
#pragma once
#include "common.cuh"
#include "neighborhood_hash.cuh"

namespace gk {

// Level j's key of every (vertex, dimension) entry e = v * d + q of one embedding set; valid[e] = 0 for q >= the
// graph's column count (no histogram row) and for a vertex the base kernel does not see (skip[v] != 0, may be null).
// u * 2^j is exact (a power-of-two scaling), so floor gives the reference's cell; gk_pm_features has checked that
// every used u lies in [0, 1 + 2^-(L-1)) (no cell beyond the clamp) and that row << j fits 64 bits.
__global__ void __launch_bounds__(256)
pm_cells(int M, int d, int j, const double* __restrict__ U, const int* __restrict__ n_cols,
         const int* __restrict__ vgraph, const int* __restrict__ labels, const unsigned char* __restrict__ skip,
         unsigned long long* __restrict__ keys, unsigned char* __restrict__ valid) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= M) return;
  const int v = e / d, q = e - v * d;
  if (q >= n_cols[vgraph[v]] || (skip && skip[v])) {
    keys[e] = 0ULL;
    valid[e] = 0;
    return;
  }
  const unsigned long long k = 1ULL << j;
  unsigned long long T = (unsigned long long)floor(__dmul_rn(U[e], (double)k));
  if (T == k) T = k - 1;
  const unsigned long long row = labels ? (unsigned long long)labels[v] * (unsigned)d + (unsigned)q : (unsigned long long)q;
  keys[e] = (row << j) | T;
  valid[e] = 1;
}

// The reference's combine (pyramid_match.py:266-285), operation for operation:
//   k = 0; for p < L: intersec[p] = I_p; k += intersec[L-1]; for q < L-1: k += 2^-(L-q-1) (intersec[q] - intersec[q+1])
// with both statements inside the level loop, so k sums L passes over a partially filled intersec (entries > p are 0).
// Every product is exact (a power of two times an integer difference); the additions round as the reference's do.
template <class Load>
__device__ __forceinline__ double pm_replay(int L, Load I) {
  double k = 0.0;
  for (int p = 0; p < L; ++p) {
    k = __dadd_rn(k, p == L - 1 ? I(L - 1) : 0.0);
    double cur = I(0);
    for (int q = 0; q < L - 1; ++q) {
      const double a = q <= p ? cur : 0.0;
      const double b = q + 1 <= p ? I(q + 1) : 0.0;
      k = __dadd_rn(k, __dmul_rn(ldexp(1.0, -(L - q - 1)), __dsub_rn(a, b)));
      cur = b;
    }
  }
  return k;
}

constexpr int PM_TILE = 32;

struct PmCombineParams {
  const float* C;    // S * L count matrices [rows x ldc], block s * L + j at C + (s * L + j) * stride
  long long stride, ldc;
  int S, L;
  int rows, cols;    // the block's rows and columns
  int mirror;        // full square matrix: upper tiles only, transposed through shared memory
  double* out;
  long long ld;
};

// K of one entry: the replayed value of every embedding set, summed in set order (WL-PM: np.sum over the levels)
__device__ __forceinline__ double pm_value(const PmCombineParams& p, long long off) {
  double s = 0.0;
  for (int t = 0; t < p.S; ++t) {
    const float* c = p.C + (long long)t * p.L * p.stride + off;
    const double k = pm_replay(p.L, [&](int j) { return (double)c[(long long)j * p.stride]; });
    s = t == 0 ? k : __dadd_rn(s, k);
  }
  return s;
}

__global__ void __launch_bounds__(PM_TILE * 8)
pm_combine(PmCombineParams p) {
  __shared__ double s_t[PM_TILE][PM_TILE + 1];
  const int nbj = (p.cols + PM_TILE - 1) / PM_TILE;
  int ti, tj;
  if (p.mirror) {  // upper-triangle tile index -> (ti, tj), tj >= ti
    long long t = blockIdx.x;
    ti = 0;
    while (t >= nbj - ti) { t -= nbj - ti; ++ti; }
    tj = ti + (int)t;
  } else {
    ti = blockIdx.x / nbj;
    tj = blockIdx.x % nbj;
  }
  const int tx = threadIdx.x & (PM_TILE - 1), ty = threadIdx.x / PM_TILE;
  const int j = tj * PM_TILE + tx;
  for (int k = ty; k < PM_TILE; k += 8) {
    const int i = ti * PM_TILE + k;
    if (i >= p.rows || j >= p.cols) continue;
    const double x = pm_value(p, (long long)i * p.ldc + j);
    p.out[(long long)i * p.ld + j] = x;
    if (p.mirror) s_t[k][tx] = x;
  }
  if (!p.mirror || ti == tj) return;
  __syncthreads();
  for (int k = ty; k < PM_TILE; k += 8) {
    const int r = tj * PM_TILE + k, c = ti * PM_TILE + tx;
    if (r < p.rows && c < p.cols) p.out[(long long)r * p.ld + c] = s_t[tx][k];
  }
}

// Self similarities: every level's self intersection is the graph's entry count m = n * n_cols (all of its rows,
// also those of labels unseen at fit; n counts the vertices that are not skipped), replayed and summed over the sets
// like pm_value.
__global__ void __launch_bounds__(256)
pm_diag(int N, int S, int L, const int* __restrict__ graph_ptr, const int* __restrict__ n_cols,
        const unsigned char* __restrict__ skip, double* __restrict__ diag) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= N) return;
  int n = graph_ptr[g + 1] - graph_ptr[g];
  if (skip)
    for (int v = graph_ptr[g]; v < graph_ptr[g + 1]; ++v) n -= skip[v] ? 1 : 0;
  double s = 0.0;
  for (int t = 0; t < S; ++t) {
    const double m = (double)((long long)n * n_cols[(long long)t * N + g]);
    const double k = pm_replay(L, [&](int) { return m; });
    s = t == 0 ? k : __dadd_rn(s, k);
  }
  diag[g] = s;
}

}  // namespace gk
