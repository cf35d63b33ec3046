// MultiscaleLaplacian (multiscale_laplacian.py; Kondor & Pan 2016): the feature-space Laplacian graph (FLG) kernel,
// fp64 throughout.  Every matrix factored here is SPD by construction on the route's scope (symmetric adjacency with
// non-negative weights, gamma > 0, heta > 0): a neighbourhood Laplacian + heta I, U^T M U + gamma I with M SPD, and the
// sum of two SPD inverses.  So Cholesky replaces the reference's general inv / eigvals; a non-positive or non-finite
// pivot still sets bit 0 of *err instead of returning a NaN.
//
//   ml_dense_adj / ml_ball1 / ml_ball_next : dense per-graph adjacency from the packed CSR, radius-l balls as 128-bit
//                                            masks (graphs of at most ML_NMAX vertices); the radius of level l is
//                                            2^(l-1), as in the reference
//   ml_vertex_C  : one CTA per (vertex, level) or per graph: Laplacian of the neighbourhood (or of the whole graph) +
//                  heta I, its Cholesky factor R, Y = R^-1 U, S = Y^T Y + gamma I, S = T T^T, the record
//                  (S^-1 = T^-T T^-1, log det S) -- the reference's calculate_C and final S
//   ml_flg_*     : one warp per (record, record) pair: Cholesky of S_a^-1 + S_b^-1, the reference's logr and its
//                  `< -30 -> 0` rule
//   ml_matmul    : U <- U Q (phi ksi at level 0, K_proj Q at the others)
#pragma once
#include "common.cuh"
#include "random_walk.cuh"  // rw_pair_of: the pair numbering of the per-pair fp64 Gram routes

namespace gk {

constexpr int ML_NMAX = 128;         // vertices of a graph: its balls are two 64-bit words
constexpr int ML_MMAX = ML_NMAX + 1; // a level-1 neighbourhood lists a vertex with a self-loop twice
constexpr int ML_PMAX = 32;          // feature width P': one warp lane per row of a P' x P' factor
constexpr int ML_NSMAX = 1024;       // vertex samples per level
constexpr int ML_THREADS = 128;
constexpr int ML_FLG_WARPS = 8;

// Bit 0 of *err: a non-positive or non-finite pivot.  Bit 1: the adjacency is not symmetric.
__device__ __forceinline__ void ml_flag(unsigned* err, unsigned bit) { atomicOr(err, bit); }

// adj[adj_off[g] + i n + j] = weight of the packed edge (i, j) of graph g (1 without weights); adj is zeroed first.
__global__ void ml_dense_adj(int V, const int* __restrict__ graph_ptr, const int* __restrict__ vgraph,
                             const int* __restrict__ row_ptr, const int* __restrict__ col_idx,
                             const double* __restrict__ w, const long long* __restrict__ adj_off, double* adj) {
  for (int u = blockIdx.x * blockDim.x + threadIdx.x; u < V; u += gridDim.x * blockDim.x) {
    const int g = vgraph[u], v0 = graph_ptr[g], n = graph_ptr[g + 1] - v0;
    double* row = adj + adj_off[g] + (long long)(u - v0) * n;
    for (int e = row_ptr[u]; e < row_ptr[u + 1]; ++e) row[col_idx[e] - v0] = w ? w[e] : 1.0;
  }
}

// Level-1 balls {u} + {j : A[u][j] > 0} (graph.py neighbors: entries > 0) and the symmetry check of A.
__global__ void ml_ball1(int V, const int* __restrict__ graph_ptr, const int* __restrict__ vgraph,
                         const long long* __restrict__ adj_off, const double* __restrict__ adj,
                         unsigned long long* ball, unsigned* err) {
  for (int u = blockIdx.x * blockDim.x + threadIdx.x; u < V; u += gridDim.x * blockDim.x) {
    const int g = vgraph[u], v0 = graph_ptr[g], n = graph_ptr[g + 1] - v0, i = u - v0;
    const double* A = adj + adj_off[g];
    unsigned long long m0 = 0, m1 = 0;
    for (int j = 0; j < n; ++j) {
      const double a = A[(long long)i * n + j];
      if (a != A[(long long)j * n + i]) ml_flag(err, 2u);
      if (a > 0.0 || j == i) {
        if (j < 64) m0 |= 1ULL << j; else m1 |= 1ULL << (j - 64);
      }
    }
    ball[2 * (long long)u] = m0;
    ball[2 * (long long)u + 1] = m1;
  }
}

// ball_{l+1}(u) = union of ball_l(w) over w in ball_l(u): graph.py produce_neighborhoods unites the level-l lists of
// the level-l neighbours, so the radius doubles from level to level (1, 2, 4, 8, ...).
__global__ void ml_ball_next(int V, const int* __restrict__ graph_ptr, const int* __restrict__ vgraph,
                             const unsigned long long* __restrict__ prev, unsigned long long* next) {
  for (int u = blockIdx.x * blockDim.x + threadIdx.x; u < V; u += gridDim.x * blockDim.x) {
    const int v0 = graph_ptr[vgraph[u]];
    const unsigned long long p[2] = {prev[2 * (long long)u], prev[2 * (long long)u + 1]};
    unsigned long long m0 = 0, m1 = 0;
    for (int h = 0; h < 2; ++h)
      for (unsigned long long b = p[h]; b; b &= b - 1) {
        const long long w = v0 + h * 64 + __ffsll((long long)b) - 1;
        m0 |= prev[2 * w];
        m1 |= prev[2 * w + 1];
      }
    next[2 * (long long)u] = m0;
    next[2 * (long long)u + 1] = m1;
  }
}

// In-place lower Cholesky of the n x n matrix A (row-major, leading dimension n) by the whole CTA; log det A into
// *logdet (thread 0's sum, in pivot order).  Returns false on a non-positive or non-finite pivot (every thread).
__device__ bool ml_chol_cta(double* A, int n, double* logdet, int* bad) {
  if (threadIdx.x == 0) { *bad = 0; *logdet = 0.0; }
  __syncthreads();
  for (int k = 0; k < n; ++k) {
    if (threadIdx.x == 0) {
      const double p = A[k * n + k];
      if (!(p > 0.0) || !isfinite(p)) *bad = 1;
      const double d = sqrt(p);
      A[k * n + k] = d;
      *logdet += 2.0 * log(d);
    }
    __syncthreads();
    if (*bad) return false;
    const double d = A[k * n + k];
    for (int i = k + 1 + threadIdx.x; i < n; i += blockDim.x) A[i * n + k] /= d;
    __syncthreads();
    const int r = n - k - 1;
    for (int t = threadIdx.x; t < r * r; t += blockDim.x) {
      const int i = k + 1 + t / r, j = k + 1 + t % r;
      if (j <= i) A[i * n + j] -= A[i * n + k] * A[j * n + k];
    }
    __syncthreads();
  }
  return true;
}

// B <- R^-1 B for the lower factor R (n x n, leading dimension n) and B n x c (leading dimension c), by the CTA.
__device__ void ml_trsm_cta(const double* R, int n, double* B, int c) {
  for (int k = 0; k < n; ++k) {
    const double d = R[k * n + k];
    for (int j = threadIdx.x; j < c; j += blockDim.x) B[k * c + j] /= d;
    __syncthreads();
    const int r = n - k - 1;
    for (int t = threadIdx.x; t < r * c; t += blockDim.x) {
      const int i = k + 1 + t / c, j = t % c;
      B[i * c + j] -= R[i * n + k] * B[k * c + j];
    }
    __syncthreads();
  }
}

struct MlUnits {
  const int* graph_ptr;
  const int* vgraph;
  const long long* adj_off;
  const double* adj;
  const unsigned long long* ball;  // [V][2] masks of this level; null: every unit is a whole graph
  int dup_loops;                   // level 1: a vertex with a self-loop is listed twice
  const double* U;                 // [V][P] features of the previous level
  int P;
  double gamma, heta;
  int n_units;
  double* rec;                     // [n_units][P P + 1]: S^-1 row-major, then log det S
  unsigned* err;
};

// One CTA per unit (grid-stride).  Shared memory: nb [ML_MMAX] int | A [max(m^2, P^2)] | Y [m P] | Z [P P], m the
// largest neighbourhood of the launch (mcap).
__global__ void __launch_bounds__(ML_THREADS) ml_vertex_C(MlUnits p, int mcap) {
  extern __shared__ double ml_smem[];
  __shared__ int nb[ML_MMAX];
  __shared__ int s_m, s_bad;
  __shared__ double s_ld, s_ld2;
  const int P = p.P;
  double* A = ml_smem;
  double* Y = A + max(mcap * mcap, P * P);
  double* Z = Y + mcap * P;
  for (int unit = blockIdx.x; unit < p.n_units; unit += gridDim.x) {
    const int g = p.ball ? p.vgraph[unit] : unit;
    const int v0 = p.graph_ptr[g], n = p.graph_ptr[g + 1] - v0;
    const double* Ag = p.adj + p.adj_off[g];
    if (threadIdx.x == 0) {
      int m = 0;
      if (p.ball) {
        const int i = unit - v0;
        for (int h = 0; h < 2; ++h)
          for (unsigned long long b = p.ball[2 * (long long)unit + h]; b; b &= b - 1) nb[m++] = h * 64 + __ffsll((long long)b) - 1;
        if (p.dup_loops && Ag[(long long)i * n + i] > 0.0) nb[m++] = i;
      } else {
        for (int i = 0; i < n; ++i) nb[i] = i;
        m = n;
      }
      s_m = m;
    }
    __syncthreads();
    const int m = s_m;
    // Laplacian of the induced matrix (its diagonal ignored, degrees from column sums, as scipy's laplacian) + heta I
    for (int t = threadIdx.x; t < m * m; t += blockDim.x) {
      const int a = t / m, b = t % m;
      A[t] = a == b ? 0.0 : -Ag[(long long)nb[a] * n + nb[b]];
    }
    __syncthreads();
    for (int b = threadIdx.x; b < m; b += blockDim.x) {
      double d = 0.0;
      for (int a = 0; a < m; ++a) d -= A[a * m + b];
      A[b * m + b] = d + p.heta;
    }
    for (int t = threadIdx.x; t < m * P; t += blockDim.x) Y[t] = p.U[(long long)(v0 + nb[t / P]) * P + t % P];
    __syncthreads();
    bool ok = ml_chol_cta(A, m, &s_ld, &s_bad);
    if (ok) {
      ml_trsm_cta(A, m, Y, P);  // Y = R^-1 U: U^T (L + heta I)^-1 U = Y^T Y
      for (int t = threadIdx.x; t < P * P; t += blockDim.x) {
        const int a = t / P, b = t % P;
        double s = 0.0;
        for (int i = 0; i < m; ++i) s += Y[i * P + a] * Y[i * P + b];
        A[t] = s + (a == b ? p.gamma : 0.0);
        Z[t] = a == b ? 1.0 : 0.0;
      }
      __syncthreads();
      ok = ml_chol_cta(A, P, &s_ld2, &s_bad);
    }
    double* out = p.rec + (long long)unit * (P * P + 1);
    if (ok) {
      ml_trsm_cta(A, P, Z, P);  // Z = T^-1, S^-1 = Z^T Z
      for (int t = threadIdx.x; t < P * P; t += blockDim.x) {
        const int a = t / P, b = t % P;
        double s = 0.0;
        for (int k = 0; k < P; ++k) s += Z[k * P + a] * Z[k * P + b];
        out[t] = s;
      }
      if (threadIdx.x == 0) out[P * P] = s_ld2;
    } else if (threadIdx.x == 0) {
      ml_flag(p.err, 1u);
      out[P * P] = nan("");
    }
    __syncthreads();  // the next unit overwrites nb and the matrices
  }
}

// FLG value of records a and b (pairwise_operation): one warp, lane i owns row i of M = S_a^-1 + S_b^-1 in `M`
// (P x P, this warp's slice of shared memory).  Every lane returns the value.
__device__ double ml_flg_warp(const double* __restrict__ ra, const double* __restrict__ rb, int P, double* M,
                              unsigned* err) {
  const int lane = threadIdx.x & 31;
  for (int t = lane; t < P * P; t += 32) M[t] = ra[t] + rb[t];
  __syncwarp();
  double ld = 0.0;
  bool bad = false;
  for (int k = 0; k < P; ++k) {
    const double p = M[k * P + k];
    if (!(p > 0.0) || !isfinite(p)) { bad = true; break; }
    const double d = sqrt(p);
    ld += 2.0 * log(d);
    const int i = lane;
    if (i > k && i < P) M[i * P + k] /= d;
    __syncwarp();
    if (i > k && i < P) {
      const double lik = M[i * P + k];
      for (int j = k + 1; j <= i; ++j) M[i * P + j] -= lik * M[j * P + k];
    }
    __syncwarp();
  }
  if (bad) {
    if (lane == 0) ml_flag(err, 1u);
    return nan("");
  }
  const double logr = (-ld - 0.5 * (ra[P * P] + rb[P * P])) / 2.0;
  return logr < -30.0 ? 0.0 : exp(logr);
}

// Projection block of one level: out[v][m] = flg(sample record m, vertex record v) for v < V, m < ns.
__global__ void __launch_bounds__(32 * ML_FLG_WARPS) ml_flg_project(const double* __restrict__ samp,
                                                                   const double* __restrict__ rec, int P, long long V,
                                                                   int ns, double* out, unsigned* err) {
  extern __shared__ double ml_smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  double* M = ml_smem + warp * P * P;
  const long long stride = P * P + 1;
  const long long n_pairs = V * ns;
  for (long long pi = (long long)blockIdx.x * ML_FLG_WARPS + warp; pi < n_pairs; pi += (long long)gridDim.x * ML_FLG_WARPS) {
    const long long v = pi / ns;
    const int m = (int)(pi - v * ns);
    const double k = ml_flg_warp(samp + m * stride, rec + v * stride, P, M, err);
    if (lane == 0) out[pi] = k;
    __syncwarp();
  }
}

// Gram pairs (RW_PAIRS_*, rw_pair_of): K[r][c] = flg(record gi, record gj); TRIANGLE mirrors to (c, r); DIAG writes
// out[r].
__global__ void __launch_bounds__(32 * ML_FLG_WARPS) ml_flg_gram(const double* __restrict__ rec, int P, int pairs,
                                                                long long n_pairs, int rows, int cols, int row_g0,
                                                                double* out, long long ld, unsigned* err) {
  extern __shared__ double ml_smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  double* M = ml_smem + warp * P * P;
  const long long stride = P * P + 1;
  for (long long pi = (long long)blockIdx.x * ML_FLG_WARPS + warp; pi < n_pairs; pi += (long long)gridDim.x * ML_FLG_WARPS) {
    int r, c, gi, gj;
    rw_pair_of(pairs, cols, row_g0, 0, pi, r, c, gi, gj);
    const double k = ml_flg_warp(rec + gi * stride, rec + gj * stride, P, M, err);
    if (lane == 0) {
      if (pairs == RW_PAIRS_DIAG) {
        out[r] = k;
      } else {
        out[(size_t)r * ld + c] = k;
        if (pairs == RW_PAIRS_TRIANGLE && c != r) out[(size_t)c * ld + r] = k;
      }
    }
    __syncwarp();
  }
}

// out[v][c] = sum_k U[v][k] Q[k][c] (k ascending): U V x w_in, Q w_in x w_out, out V x w_out.
__global__ void ml_matmul(long long V, int w_in, int w_out, const double* __restrict__ U, const double* __restrict__ Q,
                          double* out) {
  const long long n = V * w_out;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x) {
    const long long v = t / w_out;
    const int c = (int)(t - v * w_out);
    const double* u = U + v * w_in;
    double s = 0.0;
    for (int k = 0; k < w_in; ++k) s += u[k] * Q[(long long)k * w_out + c];
    out[t] = s;
  }
}

// dst[i][:] = src[ids[i]][:] for rows of `width` doubles.
__global__ void ml_gather_rows(int n, const int* __restrict__ ids, const double* __restrict__ src, long long width,
                               double* dst) {
  const long long total = (long long)n * width;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const long long i = t / width;
    dst[t] = src[(long long)ids[i] * width + (t - i * width)];
  }
}

}  // namespace gk
