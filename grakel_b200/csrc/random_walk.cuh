// Random walk kernels (random_walk.py: RandomWalk, RandomWalkLabeled), one CTA per graph pair, fp64 throughout.
//
// Routes (gk_rw_features selects one, gk_gram runs it over the pairs of the request):
//   RW_CG        scipy's cg(I - lamda M, 1, rtol=1e-6, maxiter=20) replayed step for step; K = sum(x)
//   RW_SERIES    sum_k c_k 1^T M^k 1 by repeated matvecs: c_k = mu_k (finite p) or lamda^k / k! (Taylor of expm)
//   RW_SPECTRAL  sum_a sum_b (q_a q'_b)^2 f(w_a w'_b) from the host eigen-data of both graphs
//
// The matvecs never form M.  With the reference's orientation (x.reshape((xs, ys), order="F"), multi_dot((Ax, X, Ay)),
// element e = u + n_i u'), the conjugate-gradient operator is
//   (M p)[u, u'] = sum_{v, v'} Ax[u, v] p[v, v'] Ay[v', u']  * [L(u) = L'(v')] [L(v) = L'(u')]   (RandomWalkLabeled)
// -- the label pair (a, b) selects Ax[u, v] with L(u) = a, L(v) = b and Ay[v', u'] with L'(v') = a, L'(u') = b, so the
// mask pairs u with v' and v with u'.  The power series sums 1^T M^k 1 of M = sum_ab kron(Ax^ab, Ay^ab) =
// D kron(Ax, Ay) D, D = diag([L(u) = L'(u')]); 1^T M^k 1 = 1^T (M^T)^k 1 and M^T walks the in-edges of both graphs
//   (M^T s)[u, u'] = sum_{v, v'} Ax[v, u] Ay[v', u'] s[v, v']  * [L(u) = L'(u')] [L(v) = L'(v')].
// Both are evaluated per output entry over the out-edges (CSR) / in-edges (transposed CSR) of the two vertices:
// m_i m_j terms per matvec, no intermediate n_i x n_j product, which keeps shared memory (the occupancy limit) at the
// iteration vectors.
//
// Reductions are a fixed shuffle tree per warp plus the warps' partials summed in warp order, so every run gives the
// same bits.  The vectors live in shared memory while they fit (RW_SMEM_MAX); larger pairs use a global workspace of
// the same layout, one slice per CTA.
#pragma once
#include "common.cuh"

namespace gk {

constexpr int RW_THREADS = 256;
constexpr int RW_WARPS = RW_THREADS / 32;
constexpr int RW_CG_MAXITER = 20;     // random_walk.py: cg(..., maxiter=20)
constexpr int RW_TAYLOR_CAP = 2000;   // Taylor terms before a pair is reported in rw_cap_hits
constexpr size_t RW_SMEM_MAX = 227 * 1024 - 1024;  // dynamic shared memory of one CTA (sm_90a opt-in)

enum { RW_ROUTE_CG = 0, RW_ROUTE_SPECTRAL = 1, RW_ROUTE_SERIES = 2 };
enum { RW_FN_FINITE = 0, RW_FN_EXP = 1, RW_FN_INV = 2 };
enum { RW_PAIRS_RECT = 0, RW_PAIRS_TRIANGLE = 1, RW_PAIRS_DIAG = 2 };

struct RwParams {
  const int* graph_ptr;
  const int* row_ptr; const int* col_idx; const double* val;     // out-edges (packed CSR) with their values
  const int* trow_ptr; const int* tcol_idx; const double* tval;  // in-edges (transposed CSR)
  const int* labels;                                            // vertex label ids (RandomWalkLabeled) or nullptr
  const double* q; const double* w;                             // spectral: graph g's eigen-data at graph_ptr[g]
  const double* coef; int n_coef;                               // mu_0 .. mu_p
  double lamda;
  int route, fn;
  int pairs;            // RW_PAIRS_*
  int ordered;          // 1: rows and columns index the same graphs, a pair is evaluated as op(min, max)
  long long n_pairs;
  int row_g0, rows, cols;
  double* out; long long ld;           // K rows of the request (RECT / TRIANGLE) or per-graph diagonal (DIAG)
  unsigned char* iters;                // [rows x cols] CG iterations / series terms (nullptr for DIAG)
  double* ws; long long ws_stride;     // global workspace (doubles per CTA) or nullptr: shared memory
  unsigned long long* cap_hits;
};

__device__ __forceinline__ double rw_warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Sum of NV <= 2 values over the CTA in a fixed order; `red` holds two halves of 2 x RW_WARPS doubles, used
// alternately, so one barrier per call is enough.
template <int NV>
__device__ __forceinline__ void rw_block_sum(double (&v)[NV], double* red, int& parity) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double* b = red + parity * 2 * RW_WARPS;
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    v[k] = rw_warp_sum(v[k]);
    if (lane == 0) b[k * RW_WARPS + warp] = v[k];
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    double s = 0.0;
#pragma unroll
    for (int i = 0; i < RW_WARPS; ++i) s += b[k * RW_WARPS + i];
    v[k] = s;
  }
  parity ^= 1;
}

// (M p)[e] of the conjugate-gradient operator (cross mask) at e = u + ni u'
__device__ __forceinline__ double rw_matvec_cg(const RwParams& P, int a0, int b0, int ni, int u, int up, const double* p) {
  const int* lab = P.labels;
  const int lu = lab ? lab[a0 + u] : 0, lup = lab ? lab[b0 + up] : 0;
  const int kb0 = P.trow_ptr[b0 + up], kb1 = P.trow_ptr[b0 + up + 1];
  double acc = 0.0;
  for (int ka = P.row_ptr[a0 + u], ka1 = P.row_ptr[a0 + u + 1]; ka < ka1; ++ka) {
    const int v = P.col_idx[ka] - a0;
    if (lab && lab[a0 + v] != lup) continue;
    const double av = P.val[ka];
    double s = 0.0;
    for (int kb = kb0; kb < kb1; ++kb) {
      const int vp = P.tcol_idx[kb] - b0;
      if (lab && lab[b0 + vp] != lu) continue;
      s += P.tval[kb] * p[v + ni * vp];
    }
    acc += av * s;
  }
  return acc;
}

// (M^T s)[e] of the power series (straight mask) at e = u + ni u'
__device__ __forceinline__ double rw_matvec_series(const RwParams& P, int a0, int b0, int ni, int u, int up, const double* s) {
  const int* lab = P.labels;
  if (lab && lab[a0 + u] != lab[b0 + up]) return 0.0;
  const int kb0 = P.trow_ptr[b0 + up], kb1 = P.trow_ptr[b0 + up + 1];
  double acc = 0.0;
  for (int ka = P.trow_ptr[a0 + u], ka1 = P.trow_ptr[a0 + u + 1]; ka < ka1; ++ka) {
    const int v = P.tcol_idx[ka] - a0;
    const int lv = lab ? lab[a0 + v] : 0;
    const double av = P.tval[ka];
    double t = 0.0;
    for (int kb = kb0; kb < kb1; ++kb) {
      const int vp = P.tcol_idx[kb] - b0;
      if (lab && lab[b0 + vp] != lv) continue;
      t += P.tval[kb] * s[v + ni * vp];
    }
    acc += av * t;
  }
  return acc;
}

// scipy.sparse.linalg.cg (scipy 1.18, iterative.py) on (I - lamda M) x = 1 with x0 = 0, rtol = 1e-6, maxiter = 20:
// the norm test at the top of every iteration, then beta / p / alpha / x / r in scipy's order.  sum(x) is carried as
// sum_k alpha_k 1^T p_k (x0 = 0 and x += alpha p), so x itself needs no storage.
__device__ double rw_pair_cg(const RwParams& P, int gi, int gj, double* buf, double* red, int& parity, int* iters) {
  const int a0 = P.graph_ptr[gi], ni = P.graph_ptr[gi + 1] - a0;
  const int b0 = P.graph_ptr[gj], nj = P.graph_ptr[gj + 1] - b0;
  const int mn = ni * nj;
  *iters = 0;
  if (mn == 0) return 0.0;  // sum of an empty solution
  double* r = buf;
  double* p = buf + mn;
  double* q = buf + 2 * (size_t)mn;
  const double atol = 1.0e-6 * sqrt((double)mn);  // rtol * ||b||, b = ones(mn)
  for (int e = threadIdx.x; e < mn; e += RW_THREADS) r[e] = 1.0;
  double rho = (double)mn, rho_prev = 0.0, xsum = 0.0;
  int it = 0;
  for (; it < RW_CG_MAXITER; ++it) {
    if (sqrt(rho) < atol) break;
    const double beta = it > 0 ? rho / rho_prev : 0.0;
    for (int e = threadIdx.x; e < mn; e += RW_THREADS) p[e] = it > 0 ? p[e] * beta + r[e] : r[e];
    __syncthreads();
    double pq[2] = {0.0, 0.0};
    for (int e = threadIdx.x; e < mn; e += RW_THREADS) {
      const int u = e % ni, up = e / ni;
      const double pe = p[e];
      const double qe = pe - P.lamda * rw_matvec_cg(P, a0, b0, ni, u, up, p);
      q[e] = qe;
      pq[0] += pe * qe;
      pq[1] += pe;
    }
    rw_block_sum<2>(pq, red, parity);
    const double alpha = rho / pq[0];
    xsum += alpha * pq[1];
    double rr[1] = {0.0};
    for (int e = threadIdx.x; e < mn; e += RW_THREADS) {
      const double re = r[e] - alpha * q[e];
      r[e] = re;
      rr[0] += re * re;
    }
    rw_block_sum<1>(rr, red, parity);
    rho_prev = rho;
    rho = rr[0];
  }
  *iters = it;
  return xsum;
}

// Largest row sum of a graph's (non-negative) adjacency: bounds the growth of the Taylor terms
__device__ double rw_max_row_sum(const RwParams& P, int g, double* red, int& parity) {
  const int a0 = P.graph_ptr[g], n = P.graph_ptr[g + 1] - a0;
  double m = 0.0;
  for (int u = threadIdx.x; u < n; u += RW_THREADS) {
    double s = 0.0;
    for (int k = P.row_ptr[a0 + u]; k < P.row_ptr[a0 + u + 1]; ++k) s += P.val[k];
    m = fmax(m, s);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
  double* b = red + parity * 2 * RW_WARPS;
  if ((threadIdx.x & 31) == 0) b[threadIdx.x >> 5] = m;
  __syncthreads();
  m = 0.0;
  for (int i = 0; i < RW_WARPS; ++i) m = fmax(m, b[i]);
  parity ^= 1;
  return m;
}

// sum_k c_k 1^T M^k 1.  Finite p: c_k = coef[k], k <= p, the vector s_k = M^k 1.  Taylor (fn == RW_FN_EXP):
// c_k = lamda^k / k! is carried in the vector, s_k = (lamda / k) M^T s_{k-1}, and the term is 1^T s_k.  M^k 1 alone
// grows like rho(M)^k and overflows on a hub graph while lamda^k / k! underflows, long before the stopping bound
// (0 * inf = NaN); s_k stays finite whenever the sum is.  The series stops once k >= 2 lamda R_i R_j (R = largest row
// sum; every later term is then at most half the one before, as 1^T s_{k+1} <= lamda R_i R_j / (k + 1) 1^T s_k for
// non-negative M) and the term is below 2^-56 of the partial sum, or once s_k underflows to 0.
__device__ double rw_pair_series(const RwParams& P, int gi, int gj, double* buf, double* red, int& parity, int* iters) {
  const int a0 = P.graph_ptr[gi], ni = P.graph_ptr[gi + 1] - a0;
  const int b0 = P.graph_ptr[gj], nj = P.graph_ptr[gj + 1] - b0;
  const int mn = ni * nj;
  *iters = 0;
  if (mn == 0) return 0.0;
  double* s = buf;
  double* t = buf + mn;
  for (int e = threadIdx.x; e < mn; e += RW_THREADS) s[e] = 1.0;
  const bool taylor = P.fn == RW_FN_EXP;
  double kmin = 0.0;
  if (taylor) kmin = 2.0 * P.lamda * rw_max_row_sum(P, gi, red, parity) * rw_max_row_sum(P, gj, red, parity);
  double S = (taylor ? 1.0 : P.coef[0]) * (double)mn;
  const int kmax = taylor ? RW_TAYLOR_CAP : P.n_coef - 1;
  int k = 1;
  for (; k <= kmax; ++k) {
    __syncthreads();
    const double f = taylor ? P.lamda / (double)k : 1.0;
    double tot[1] = {0.0};
    for (int e = threadIdx.x; e < mn; e += RW_THREADS) {
      const double v = f * rw_matvec_series(P, a0, b0, ni, e % ni, e / ni, s);
      t[e] = v;
      tot[0] += v;
    }
    rw_block_sum<1>(tot, red, parity);
    const double term = taylor ? tot[0] : P.coef[k] * tot[0];
    S += term;
    double* x = s; s = t; t = x;
    if (taylor && (double)k >= kmin && fabs(term) < 0x1p-56 * fabs(S)) break;
    // s_k = 0 (M^k 1 = 0, or the scaled terms fell below the smallest subnormal): every later term is 0, or at most
    // that small times n_i n_j against S >= n_i n_j
    if (tot[0] == 0.0 && taylor) break;
  }
  if (taylor && k > kmax && threadIdx.x == 0) atomicAdd(P.cap_hits, 1ull);
  *iters = k > kmax ? kmax : k;
  return S;
}

// sum_a sum_b (q_a q'_b)^2 f(w_a w'_b).  The finite series runs as the reference's `D *= Dij; S += mu_k D`.
__device__ double rw_pair_spectral(const RwParams& P, int gi, int gj, double* red, int& parity) {
  const int a0 = P.graph_ptr[gi], ni = P.graph_ptr[gi + 1] - a0;
  const int b0 = P.graph_ptr[gj], nj = P.graph_ptr[gj + 1] - b0;
  const int mn = ni * nj;
  double acc[1] = {0.0};
  for (int e = threadIdx.x; e < mn; e += RW_THREADS) {
    const int a = e / nj, b = e - a * nj;
    const double ff = P.q[a0 + a] * P.q[b0 + b];
    const double z = P.w[a0 + a] * P.w[b0 + b];
    double S;
    if (P.fn == RW_FN_FINITE) {
      double D = 1.0;
      S = P.coef[0] * D;
      for (int k = 1; k < P.n_coef; ++k) {
        D *= z;
        S += P.coef[k] * D;
      }
    } else if (P.fn == RW_FN_EXP) {
      S = exp(P.lamda * z);
    } else {
      S = 1.0 / (1.0 - P.lamda * z);
    }
    acc[0] += ff * S * ff;
  }
  rw_block_sum<1>(acc, red, parity);
  return acc[0];
}

// Entry (r, c) of pair number pi and the graphs (gi, gj) it is evaluated on.  RECT: entry (r, c) of the request;
// TRIANGLE: the upper triangle of the square case (the caller mirrors it to (c, r)); DIAG: graph r against itself.
// `ordered`: rows and columns index the same graphs and the pair is evaluated as op(min, max).
__device__ __forceinline__ void rw_pair_of(int pairs, int cols, int row_g0, int ordered, long long pi, int& r, int& c,
                                           int& gi, int& gj) {
  if (pairs == RW_PAIRS_TRIANGLE) {
    // row r holds cols - r entries starting at r cols - r (r - 1) / 2
    const double n = (double)cols;
    r = (int)floor(((2.0 * n + 1.0) - sqrt((2.0 * n + 1.0) * (2.0 * n + 1.0) - 8.0 * (double)pi)) * 0.5);
    r = max(0, min(r, cols - 1));
    auto start = [&](long long rr) { return rr * (long long)cols - rr * (rr - 1) / 2; };
    while (r > 0 && start(r) > pi) --r;
    while (r + 1 < cols && start(r + 1) <= pi) ++r;
    c = r + (int)(pi - start(r));
  } else if (pairs == RW_PAIRS_DIAG) {
    r = c = (int)pi;
  } else {
    r = (int)(pi / cols);
    c = (int)(pi - (long long)r * cols);
  }
  gi = pairs == RW_PAIRS_DIAG ? r : row_g0 + r;
  gj = c;
  if (ordered && gi > gj) { const int x = gi; gi = gj; gj = x; }
}

// One CTA per pair (grid-stride), written to (r, c) of the request and, for TRIANGLE, mirrored to (c, r).
__global__ void __launch_bounds__(RW_THREADS) rw_pairs(RwParams P) {
  extern __shared__ double rw_smem[];
  __shared__ double red[2 * 2 * RW_WARPS];
  double* buf = P.ws ? P.ws + (size_t)blockIdx.x * P.ws_stride : rw_smem;
  int parity = 0;
  for (long long pi = blockIdx.x; pi < P.n_pairs; pi += gridDim.x) {
    int r, c, gi, gj;
    rw_pair_of(P.pairs, P.cols, P.row_g0, P.ordered, pi, r, c, gi, gj);
    int it = 0;
    double v;
    if (P.route == RW_ROUTE_CG) v = rw_pair_cg(P, gi, gj, buf, red, parity, &it);
    else if (P.route == RW_ROUTE_SERIES) v = rw_pair_series(P, gi, gj, buf, red, parity, &it);
    else v = rw_pair_spectral(P, gi, gj, red, parity);
    if (threadIdx.x == 0) {
      const unsigned char itb = (unsigned char)min(it, 255);
      if (P.pairs == RW_PAIRS_DIAG) {
        P.out[r] = v;
      } else {
        P.out[(size_t)r * P.ld + c] = v;
        if (P.iters) P.iters[(size_t)r * P.cols + c] = itb;
        if (P.pairs == RW_PAIRS_TRIANGLE && c != r) {
          P.out[(size_t)c * P.ld + r] = v;
          if (P.iters) P.iters[(size_t)c * P.cols + r] = itb;
        }
      }
    }
    __syncthreads();  // the next pair overwrites the vectors
  }
}

}  // namespace gk
