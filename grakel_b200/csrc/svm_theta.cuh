// SvmTheta (svm_theta.py): per graph, fp64 throughout,
//   svmt_eig  the smallest eigenvalue m of the 0/1 adjacency with its upper triangle mirrored (scipy's
//             eigvalsh(lower=False)): Householder tridiagonalisation in shared memory, then Sturm-count multisection,
//             one CTA per graph;
//   svmt_smo  libsvm's one-class Solver (scikit-learn's svm.cpp, Solve with shrinking, nu = 0.5, eps = 1e-3) on the
//             matrix K = (A > 1e-10) / -m with unit diagonal (or the plain 0/1 matrix when m >= -1e-6), one warp per
//             graph.  Q is never stored: an entry is the float of 0, the edge value or the diagonal value, read from the
//             row bitmask of the original vertex behind each active-set position.  Every operation the reference
//             rounds is rounded here the same way (__dmul_rn / __dadd_rn: no contraction into FMA), so the alphas and
//             the iteration counts are the reference's;
//   svmt_phi  the sampled subset sums and their level means, one warp per graph, in numpy's summation order.
// The MT19937 draws of the samples (`RandomState.choice(n, k, replace=False)`) are host code: svmt_draw.
#pragma once
#include "common.cuh"

namespace gk {

constexpr int SVMT_NMAX = 128;        // vertices per graph: the eigen workspace is n^2 doubles of shared memory
constexpr int SVMT_EIG_THREADS = 256;
constexpr int SVMT_SMO_WARPS = 4;
constexpr int SVMT_PHI_WARPS = 4;
constexpr int SVMT_STACK = 48;        // frames of the pairwise-sum recursion (depth ~ log2(n / 128))
constexpr long long SVMT_MAX_ITER = 10000000;  // SMO iterations before a graph is reported as not converging
constexpr double SVMT_TAU = 1e-12;
constexpr double SVMT_EPS = 1e-3;

enum : unsigned { SVMT_ERR_ITER = 1u, SVMT_ERR_INDEX = 2u };
enum : unsigned char { SVMT_LOWER = 0, SVMT_UPPER = 1, SVMT_FREE = 2 };

// ------------------------------------------------------------------ smallest eigenvalue
__device__ __forceinline__ double svmt_block_sum(double v, double* red) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
  for (int w = 0; w < SVMT_EIG_THREADS / 32; ++w) s += red[w];
  return s;
}

// Eigenvalues of the tridiagonal (d, e) below x.
__device__ __forceinline__ int svmt_sturm(const double* d, const double* e, int n, double x) {
  int c = 0;
  double q = d[0] - x;
  for (int i = 0;;) {
    if (fabs(q) < 1e-290) q = -1e-290;
    c += q < 0.0;
    if (++i == n) break;
    q = (d[i] - x) - e[i - 1] * e[i - 1] / q;
  }
  return c;
}

__global__ void __launch_bounds__(SVMT_EIG_THREADS)
svmt_eig(const int* __restrict__ vptr, const unsigned* __restrict__ adj, int n_graphs, double* __restrict__ m_out) {
  extern __shared__ double sm[];
  __shared__ double red[SVMT_EIG_THREADS / 32];
  __shared__ double s_lo, s_hi;
  __shared__ int s_first;
  const int tid = threadIdx.x, T = SVMT_EIG_THREADS;
  for (int g = blockIdx.x; g < n_graphs; g += gridDim.x) {
    const int v0 = vptr[g], n = vptr[g + 1] - v0;
    double* A = sm;
    double* d = A + n * n;
    double* e = d + n;
    double* v = e + n;
    double* p = v + n;
    for (int idx = tid; idx < n * n; idx += T) {
      const int i = idx / n, j = idx - i * n, a = min(i, j), b = max(i, j);
      A[idx] = (a != b && ((adj[(size_t)(v0 + a) * 4 + (b >> 5)] >> (b & 31)) & 1u)) ? 1.0 : 0.0;
    }
    __syncthreads();
    for (int k = 0; k + 2 < n; ++k) {
      double s = 0.0;
      for (int i = k + 1 + tid; i < n; i += T) s += A[i * n + k] * A[i * n + k];
      const double ss = svmt_block_sum(s, red);
      const double x0 = A[(k + 1) * n + k];
      if (ss == 0.0) {  // the column is already reduced
        if (tid == 0) { d[k] = A[k * n + k]; e[k] = 0.0; }
        __syncthreads();
        continue;
      }
      const double alpha = x0 > 0.0 ? -sqrt(ss) : sqrt(ss);
      const double hh = ss - x0 * alpha;  // v^T v / 2
      for (int i = k + 1 + tid; i < n; i += T) v[i] = i == k + 1 ? x0 - alpha : A[i * n + k];
      __syncthreads();
      for (int i = k + 1 + tid; i < n; i += T) {
        double acc = 0.0;
        for (int j = k + 1; j < n; ++j) acc += A[i * n + j] * v[j];
        p[i] = acc / hh;
      }
      __syncthreads();
      double t = 0.0;
      for (int i = k + 1 + tid; i < n; i += T) t += v[i] * p[i];
      const double kk = svmt_block_sum(t, red) / (2.0 * hh);
      for (int i = k + 1 + tid; i < n; i += T) p[i] -= kk * v[i];
      __syncthreads();
      const int r = n - k - 1;
      for (int idx = tid; idx < r * r; idx += T) {
        const int i = k + 1 + idx / r, j = k + 1 + idx % r;
        A[i * n + j] -= v[i] * p[j] + p[i] * v[j];
      }
      if (tid == 0) { d[k] = A[k * n + k]; e[k] = alpha; }
      __syncthreads();
    }
    if (tid == 0) {
      if (n >= 2) {
        d[n - 2] = A[(n - 2) * n + n - 2];
        d[n - 1] = A[(n - 1) * n + n - 1];
        e[n - 2] = A[(n - 1) * n + n - 2];
      } else {
        d[0] = A[0];
      }
      double lo = d[0], hi = d[0];
      for (int i = 0; i < n; ++i) {
        const double r = (i > 0 ? fabs(e[i - 1]) : 0.0) + (i + 1 < n ? fabs(e[i]) : 0.0);
        lo = fmin(lo, d[i] - r);
        hi = fmax(hi, d[i] + r);
      }
      s_lo = lo - 1e-300;
      s_hi = hi + 1e-300;
    }
    __syncthreads();
    // multisection: every thread counts at one point of (lo, hi); the first point with a count keeps the interval
    for (int round = 0; round < 64; ++round) {
      const double lo = s_lo, hi = s_hi;
      const double x = lo + (hi - lo) * ((double)(tid + 1) / (T + 1));
      if (tid == 0) s_first = T;
      __syncthreads();
      if (x > lo && x < hi && svmt_sturm(d, e, n, x) >= 1) atomicMin(&s_first, tid);
      __syncthreads();
      const int f = s_first;
      const double nlo = f == 0 ? lo : lo + (hi - lo) * ((double)f / (T + 1));
      const double nhi = f == T ? hi : lo + (hi - lo) * ((double)(f + 1) / (T + 1));
      __syncthreads();
      if (tid == 0) { s_lo = fmax(lo, nlo); s_hi = fmin(hi, nhi); }
      __syncthreads();
      if (s_lo == lo && s_hi == hi) break;
    }
    if (tid == 0) m_out[g] = 0.5 * (s_lo + s_hi);
    __syncthreads();
  }
}

// ------------------------------------------------------------------ one-class SMO
struct SvmtWarp {
  double G[SVMT_NMAX], Gb[SVMT_NMAX], al[SVMT_NMAX];
  unsigned rows[SVMT_NMAX][4];  // out-edge bitmask of each original vertex
  unsigned char perm[SVMT_NMAX], st[SVMT_NMAX];
};

struct SvmtQ {
  float qe, qd;  // Qfloat of an edge and of the diagonal
  double QD;
};

__device__ __forceinline__ float svmt_q(const SvmtWarp& w, const SvmtQ& q, int i, int k) {
  if (i == k) return q.qd;
  const int a = w.perm[i], b = w.perm[k];
  return ((w.rows[a][b >> 5] >> (b & 31)) & 1u) ? q.qe : 0.0f;
}

__device__ __forceinline__ unsigned char svmt_status(double a) {
  return a >= 1.0 ? SVMT_UPPER : a <= 0.0 ? SVMT_LOWER : SVMT_FREE;
}

// (value, index) of the sequential `if (x >= best)` scan: the largest value, the last index among equals
__device__ __forceinline__ void svmt_argmax(double& v, int& i) {
  for (int o = 16; o > 0; o >>= 1) {
    const double ov = __shfl_xor_sync(0xffffffffu, v, o);
    const int oi = __shfl_xor_sync(0xffffffffu, i, o);
    if (ov > v || (ov == v && oi > i)) { v = ov; i = oi; }
  }
}

// the sequential `if (x <= best)` scan: the smallest value, the last index among equals
__device__ __forceinline__ void svmt_argmin(double& v, int& i) {
  for (int o = 16; o > 0; o >>= 1) {
    const double ov = __shfl_xor_sync(0xffffffffu, v, o);
    const int oi = __shfl_xor_sync(0xffffffffu, i, o);
    if (ov < v || (ov == v && oi > i)) { v = ov; i = oi; }
  }
}

__device__ __forceinline__ double svmt_max(double v) {
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Solver::reconstruct_gradient
__device__ __forceinline__ void svmt_reconstruct(SvmtWarp& w, const SvmtQ& q, int l, int active, int lane) {
  if (active == l) return;
  for (int j = active + lane; j < l; j += 32) w.G[j] = __dadd_rn(w.Gb[j], 0.0);
  int nr_free = 0;
  for (int j0 = 0; j0 < active; j0 += 32) {
    const int j = j0 + lane;
    nr_free += __popc(__ballot_sync(0xffffffffu, j < active && w.st[j] == SVMT_FREE));
  }
  __syncwarp();
  if ((long long)nr_free * l > 2LL * active * (l - active)) {
    for (int i = active + lane; i < l; i += 32) {
      double gi = w.G[i];
      for (int j = 0; j < active; ++j)
        if (w.st[j] == SVMT_FREE) gi = __dadd_rn(gi, __dmul_rn(w.al[j], (double)svmt_q(w, q, i, j)));
      w.G[i] = gi;
    }
  } else {
    for (int j = active + lane; j < l; j += 32) {
      double gj = w.G[j];
      for (int i = 0; i < active; ++i)
        if (w.st[i] == SVMT_FREE) gj = __dadd_rn(gj, __dmul_rn(w.al[i], (double)svmt_q(w, q, i, j)));
      w.G[j] = gj;
    }
  }
  __syncwarp();
}

// Solver::select_working_set for y = +1 everywhere: the pair (i, j), or (-1, -1) when optimal
__device__ __forceinline__ int2 svmt_select(const SvmtWarp& w, const SvmtQ& q, int active, int lane) {
  double gmax = -INFINITY;
  int gi = -1;
  for (int t = lane; t < active; t += 32)
    if (w.st[t] != SVMT_UPPER && -w.G[t] >= gmax) { gmax = -w.G[t]; gi = t; }
  svmt_argmax(gmax, gi);
  double gmax2 = -INFINITY, omin = INFINITY;
  int gj = -1;
  for (int j = lane; j < active; j += 32) {
    if (w.st[j] == SVMT_LOWER) continue;
    const double gd = __dadd_rn(gmax, w.G[j]);
    if (w.G[j] >= gmax2) gmax2 = w.G[j];
    if (gd > 0.0) {
      const double quad = __dsub_rn(__dadd_rn(q.QD, q.QD), __dmul_rn(2.0, (double)svmt_q(w, q, gi, j)));
      const double od = __ddiv_rn(-__dmul_rn(gd, gd), quad > 0.0 ? quad : SVMT_TAU);
      if (od <= omin) { omin = od; gj = j; }
    }
  }
  gmax2 = svmt_max(gmax2);
  svmt_argmin(omin, gj);
  if (__dadd_rn(gmax, gmax2) < SVMT_EPS || gj == -1) return make_int2(-1, -1);
  return make_int2(gi, gj);
}

__device__ __forceinline__ bool svmt_be_shrunk(const SvmtWarp& w, int i, double gmax1, double gmax2) {
  if (w.st[i] == SVMT_UPPER) return -w.G[i] > gmax1;
  if (w.st[i] == SVMT_LOWER) return w.G[i] > gmax2;
  return false;
}

__device__ __forceinline__ void svmt_swap(SvmtWarp& w, int i, int j) {
  double t = w.G[i]; w.G[i] = w.G[j]; w.G[j] = t;
  t = w.Gb[i]; w.Gb[i] = w.Gb[j]; w.Gb[j] = t;
  t = w.al[i]; w.al[i] = w.al[j]; w.al[j] = t;
  unsigned char c = w.st[i]; w.st[i] = w.st[j]; w.st[j] = c;
  c = w.perm[i]; w.perm[i] = w.perm[j]; w.perm[j] = c;
}

// Solver::do_shrinking; returns the new active size, negated once the gradient has been reconstructed (unshrink)
__device__ __forceinline__ int svmt_shrink(SvmtWarp& w, const SvmtQ& q, int l, int active, bool unshrink, int lane) {
  double gmax1 = -INFINITY, gmax2 = -INFINITY;
  for (int i = lane; i < active; i += 32) {
    if (w.st[i] != SVMT_UPPER) gmax1 = fmax(gmax1, -w.G[i]);
    if (w.st[i] != SVMT_LOWER) gmax2 = fmax(gmax2, w.G[i]);
  }
  gmax1 = svmt_max(gmax1);
  gmax2 = svmt_max(gmax2);
  const bool now = !unshrink && __dadd_rn(gmax1, gmax2) <= __dmul_rn(SVMT_EPS, 10.0);
  if (now) {
    svmt_reconstruct(w, q, l, active, lane);
    active = l;
  }
  if (lane == 0) {
    for (int i = 0; i < active; ++i)
      if (svmt_be_shrunk(w, i, gmax1, gmax2)) {
        active--;
        while (active > i) {
          if (!svmt_be_shrunk(w, active, gmax1, gmax2)) {
            svmt_swap(w, i, active);
            break;
          }
          active--;
        }
      }
  }
  __syncwarp();
  active = __shfl_sync(0xffffffffu, active, 0);
  return now ? -active : active;
}

__global__ void __launch_bounds__(32 * SVMT_SMO_WARPS, 4)
svmt_smo(const int* __restrict__ vptr, const unsigned* __restrict__ adj, int n_graphs, const double* __restrict__ m_in,
         double* __restrict__ alpha_out, int* __restrict__ iters_out, unsigned* __restrict__ err) {
  __shared__ SvmtWarp ws[SVMT_SMO_WARPS];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  SvmtWarp& w = ws[wid];
  for (int g = blockIdx.x * SVMT_SMO_WARPS + wid; g < n_graphs; g += gridDim.x * SVMT_SMO_WARPS) {
    const int v0 = vptr[g], l = vptr[g + 1] - v0;
    const double m = m_in[g];
    SvmtQ q;
    if (m < 0.0 && fabs(m) > 1e-6) {  // K /= -m, then the diagonal becomes 1
      q.qe = (float)__ddiv_rn(1.0, -m); q.qd = 1.0f; q.QD = 1.0;
    } else {
      q.qe = 1.0f; q.qd = 0.0f; q.QD = 0.0;
    }
    for (int k = lane; k < l; k += 32) {
      for (int c = 0; c < 4; ++c) w.rows[k][c] = adj[(size_t)(v0 + k) * 4 + c];
      // solve_one_class: nu * l = l / 2 spread over the leading alphas
      const double a = 2 * k + 2 <= l ? 1.0 : (2 * k + 1 == l ? 0.5 : 0.0);
      w.al[k] = a; w.st[k] = svmt_status(a); w.perm[k] = (unsigned char)k;
    }
    __syncwarp();
    for (int j = lane; j < l; j += 32) {  // G = Q alpha, G_bar = C Q over the alphas at the upper bound
      double gj = 0.0, bj = 0.0;
      for (int i = 0; i < l; ++i) {
        if (w.st[i] == SVMT_LOWER) continue;
        const double qij = (double)svmt_q(w, q, i, j);
        gj = __dadd_rn(gj, __dmul_rn(w.al[i], qij));
        if (w.st[i] == SVMT_UPPER) bj = __dadd_rn(bj, qij);
      }
      w.G[j] = gj; w.Gb[j] = bj;
    }
    __syncwarp();
    long long iter = 0;
    int counter = min(l, 1000) + 1, active = l;
    bool unshrink = false, failed = false;
    while (true) {
      if (--counter == 0) {
        counter = min(l, 1000);
        active = svmt_shrink(w, q, l, active, unshrink, lane);
        if (active < 0) { active = -active; unshrink = true; }
      }
      int2 ij = svmt_select(w, q, active, lane);
      if (ij.x < 0) {
        svmt_reconstruct(w, q, l, active, lane);
        active = l;
        ij = svmt_select(w, q, active, lane);
        if (ij.x < 0) break;
        counter = 1;
      }
      const int i = ij.x, j = ij.y;
      if (iter >= SVMT_MAX_ITER) { failed = true; break; }
      ++iter;
      const double old_i = w.al[i], old_j = w.al[j];
      const double quad0 = __dsub_rn(__dadd_rn(q.QD, q.QD), (double)(2.0f * svmt_q(w, q, i, j)));
      const double quad = quad0 <= 0.0 ? SVMT_TAU : quad0;
      const double delta = __ddiv_rn(__dsub_rn(w.G[i], w.G[j]), quad);
      const double sum = __dadd_rn(old_i, old_j);
      double ai = __dsub_rn(old_i, delta), aj = __dadd_rn(old_j, delta);
      if (sum > 1.0) {
        if (ai > 1.0) { ai = 1.0; aj = __dsub_rn(sum, 1.0); }
      } else if (aj < 0.0) {
        aj = 0.0; ai = sum;
      }
      if (sum > 1.0) {
        if (aj > 1.0) { aj = 1.0; ai = __dsub_rn(sum, 1.0); }
      } else if (ai < 0.0) {
        ai = 0.0; aj = sum;
      }
      const double dai = __dsub_rn(ai, old_i), daj = __dsub_rn(aj, old_j);
      const bool ui = w.st[i] == SVMT_UPPER, uj = w.st[j] == SVMT_UPPER;
      const unsigned char si = svmt_status(ai), sj = svmt_status(aj);
      __syncwarp();
      for (int k = lane; k < active; k += 32) {
        const double t = __dadd_rn(__dmul_rn((double)svmt_q(w, q, i, k), dai), __dmul_rn((double)svmt_q(w, q, j, k), daj));
        w.G[k] = __dadd_rn(w.G[k], t);
      }
      const bool fi = ui != (si == SVMT_UPPER), fj = uj != (sj == SVMT_UPPER);
      if (fi || fj) {
        for (int k = lane; k < l; k += 32) {
          double b = w.Gb[k];
          if (fi) { const double qk = (double)svmt_q(w, q, i, k); b = ui ? __dsub_rn(b, qk) : __dadd_rn(b, qk); }
          if (fj) { const double qk = (double)svmt_q(w, q, j, k); b = uj ? __dsub_rn(b, qk) : __dadd_rn(b, qk); }
          w.Gb[k] = b;
        }
      }
      __syncwarp();
      if (lane == 0) { w.al[i] = ai; w.al[j] = aj; w.st[i] = si; w.st[j] = sj; }
      __syncwarp();
    }
    for (int k = lane; k < l; k += 32) alpha_out[v0 + w.perm[k]] = w.al[k];
    if (lane == 0) {
      iters_out[g] = (int)iter;
      if (failed) atomicOr(err, SVMT_ERR_ITER);
    }
    __syncwarp();
  }
}

// ------------------------------------------------------------------ subset sums and level means
// numpy's pairwise_sum of n <= 128 values x(0) .. x(n - 1): a plain loop from -0.0 below 8, else eight accumulators
template <class X>
__device__ __forceinline__ double svmt_block(X x, int n) {
  if (n < 8) {
    double r = -0.0;
    for (int i = 0; i < n; ++i) r = __dadd_rn(r, x(i));
    return r;
  }
  double r[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) r[j] = x(j);
  int i = 8;
  for (; i < n - n % 8; i += 8)
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = __dadd_rn(r[j], x(i + j));
  double res = __dadd_rn(__dadd_rn(__dadd_rn(r[0], r[1]), __dadd_rn(r[2], r[3])),
                         __dadd_rn(__dadd_rn(r[4], r[5]), __dadd_rn(r[6], r[7])));
  for (; i < n; ++i) res = __dadd_rn(res, x(i));
  return res;
}

struct SvmtStack {
  long long off[SVMT_STACK], len[SVMT_STACK];
  double left[SVMT_STACK];
  int stage[SVMT_STACK];
};

// numpy's pairwise_sum of a[0 .. n): blocks of at most 128, halves split at a multiple of 8 (one thread)
__device__ __forceinline__ double svmt_pairwise(const double* a, long long n, SvmtStack& s) {
  int sp = 0;
  double ret = 0.0;
  s.off[0] = 0; s.len[0] = n; s.stage[0] = 0;
  while (sp >= 0) {
    const long long off = s.off[sp], len = s.len[sp];
    if (len <= 128) {
      ret = svmt_block([=](int i) { return a[off + i]; }, (int)len);
      --sp;
      continue;
    }
    long long n2 = len / 2;
    n2 -= n2 % 8;
    if (s.stage[sp] == 0) {
      s.stage[sp] = 1;
      ++sp; s.off[sp] = off; s.len[sp] = n2; s.stage[sp] = 0;
    } else if (s.stage[sp] == 1) {
      s.left[sp] = ret; s.stage[sp] = 2;
      ++sp; s.off[sp] = off + n2; s.len[sp] = len - n2; s.stage[sp] = 0;
    } else {
      ret = __dadd_rn(s.left[sp], ret);
      --sp;
    }
  }
  return ret;
}

// phi[g][li] = mean over the level's samples of the sum of the alphas at the drawn indexes (all n alphas for a level
// above n), 0 for a level without samples; the first level also goes to rec[g].  A drawn index outside its graph sets
// SVMT_ERR_INDEX and is not read.
__global__ void __launch_bounds__(32 * SVMT_PHI_WARPS, 4)
svmt_phi(const int* __restrict__ vptr, int n_graphs, const double* __restrict__ alpha, int lo, int L,
         const int* __restrict__ counts, const long long* __restrict__ draw_off, const unsigned char* __restrict__ idx,
         const long long* __restrict__ sum_off, double* __restrict__ sums, double* __restrict__ phi,
         double* __restrict__ rec, unsigned* __restrict__ err) {
  __shared__ SvmtStack stk[SVMT_PHI_WARPS];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int g = blockIdx.x * SVMT_PHI_WARPS + wid; g < n_graphs; g += gridDim.x * SVMT_PHI_WARPS) {
    const int v0 = vptr[g], n = vptr[g + 1] - v0;
    const double* a = alpha + v0;
    long long doff = draw_off[g], soff = sum_off[g];
    for (int li = 0; li < L; ++li) {
      const int v = counts[(size_t)g * L + li], level = lo + li;
      double mean = 0.0;
      if (v > 0) {
        double* s = sums + soff;
        if (level <= n) {
          for (int k = lane; k < v; k += 32) {
            const unsigned char* ix = idx + doff + (long long)k * level;
            bool inside = true;
            for (int i = 0; i < level; ++i) inside &= ix[i] < n;
            if (inside) {
              s[k] = svmt_block([=](int i) { return a[ix[i]]; }, level);
            } else {
              s[k] = 0.0;
              atomicOr(err, SVMT_ERR_INDEX);
            }
          }
          doff += (long long)v * level;
        } else {
          const double all = svmt_block([=](int i) { return a[i]; }, n);
          for (int k = lane; k < v; k += 32) s[k] = all;
        }
        __syncwarp();
        if (lane == 0) mean = __ddiv_rn(svmt_pairwise(s, v, stk[wid]), (double)v);
        soff += v;
      }
      if (lane == 0) {
        phi[(size_t)g * L + li] = mean;
        if (li == 0) rec[g] = mean;
      }
    }
    __syncwarp();
  }
}

__global__ void svmt_diag(const double* __restrict__ rec, long long n, double* __restrict__ diag) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    diag[i] = __dmul_rn(rec[i], rec[i]);
}

// ------------------------------------------------------------------ host: numpy's legacy RandomState draws
struct SvmtMT {
  uint32_t* key;  // 624 words
  int pos;
  uint32_t next() {
    if (pos >= 624) {
      const uint32_t UP = 0x80000000u, LO = 0x7fffffffu, MA = 0x9908b0dfu;
      int i = 0;
      for (; i < 624 - 397; ++i) {
        const uint32_t y = (key[i] & UP) | (key[i + 1] & LO);
        key[i] = key[i + 397] ^ (y >> 1) ^ (0u - (y & 1u) & MA);
      }
      for (; i < 623; ++i) {
        const uint32_t y = (key[i] & UP) | (key[i + 1] & LO);
        key[i] = key[i + 397 - 624] ^ (y >> 1) ^ (0u - (y & 1u) & MA);
      }
      const uint32_t y = (key[623] & UP) | (key[0] & LO);
      key[623] = key[396] ^ (y >> 1) ^ (0u - (y & 1u) & MA);
      pos = 0;
    }
    uint32_t y = key[pos++];
    y ^= y >> 11;
    y ^= (y << 7) & 0x9d2c5680u;
    y ^= (y << 15) & 0xefc60000u;
    y ^= y >> 18;
    return y;
  }
  // random_interval(max): masked 32-bit words, redrawn while above max
  uint32_t interval(uint32_t max) {
    if (max == 0) return 0;
    uint32_t mask = max;
    mask |= mask >> 1; mask |= mask >> 2; mask |= mask >> 4; mask |= mask >> 8; mask |= mask >> 16;
    uint32_t v;
    while ((v = (next() & mask)) > max) {
    }
    return v;
  }
  // legacy RandomState.permutation(n): arange(n) shuffled by Fisher-Yates from the top (choice(n, r, replace=False)
  // is its first r entries)
  template <class T>
  void permutation(T* perm, int n) {
    for (int i = 0; i < n; ++i) perm[i] = (T)i;
    for (int i = n - 1; i >= 1; --i) {
      const uint32_t j = interval((uint32_t)i);
      const T t = perm[i]; perm[i] = perm[j]; perm[j] = t;
    }
  }
};

}  // namespace gk
