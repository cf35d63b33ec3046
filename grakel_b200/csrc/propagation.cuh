// Propagation / PropagationAttr (Neumann et al. 2016; propagation.py:27-689) on the device.
//
// Every graph keeps a dense fp64 matrix P (V x D: one-hot labels, or the vertex attributes).  Level t hashes every
// vertex into a bin, then every graph does P <- T P with its row-normalised transition matrix T (a CSR the host
// builds with sklearn's normalize).  K = sum_t Phi_t Phi_t^T, Phi_t[g, c] the number of vertices of graph g in bin
// c at level t: the bins of every level become dense columns of their own (level after level, so levels never share
// a column) and (graph, column) counts go into the SP / WL feature table, whose exact integer Gram gk_gram runs.
//
// Numerics.  A bin is floor(x) of the reference's x = (dot(P_v, u) + b) / w (labelled) or x_j = (P_vj u_j + b_j) / w
// (attributes): every operation is one correctly rounded IEEE operation, no contraction of the "+ b", no multiply
// by 1/w.  Sums run in a fixed order (ascending column, one FMA chain from +0), which numpy's BLAS need not share, so
// a bin can differ from the reference's only when x lies within rounding distance of an integer.  Such x are
// counted (pk_near_edge): |x - rint(x)| <= 2^-30 * max(m, 1), m the magnitude of the terms of x.  Two summation
// orders, including the rounding carried in P through t earlier steps, differ by less than 2 (D + t deg + 2) 2^-53 m
// (D columns, deg the longest row of T), which is inside the margin while D + t_max deg <= 2^22 (DESIGN 4.12).  P
// stored as float32 or truncated to integers (PropagationAttr keeps the attribute dtype) has its own edges, counted
// the same way.
#pragma once
#include "common.cuh"
#include "wl.cuh"

namespace gk {

constexpr int PK_STORE_F64 = 0, PK_STORE_F32 = 1, PK_STORE_INT = 2;
constexpr double PK_MARGIN = 9.313225746154785e-10;  // 2^-30

__device__ __forceinline__ bool pk_near_int(double x, double mag) {
  return fabs(x - rint(x)) <= PK_MARGIN * fmax(mag, 1.0);
}

// level-0 P of the labelled kernel: one-hot rows (P cleared by the caller)
__global__ void __launch_bounds__(256)
pk_onehot(int V, int D, const int* __restrict__ labels, double* __restrict__ P) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v < V) P[(long long)v * D + labels[v]] = 1.0;
}

// P_out[i, c] = sum over row i's non-zeros k of T[i, k] P_in[k, c], in ascending k, then stored as fp64, rounded to
// float32 or truncated toward zero (numpy's assignment into a float32 / integer P, propagation.py:628).  One thread
// per entry, c fastest: a warp reads consecutive columns of the same neighbour rows.
__global__ void __launch_bounds__(256)
pk_propagate(long long n, int D, const int* __restrict__ row_ptr, const int* __restrict__ col_idx,
             const double* __restrict__ tval, const double* __restrict__ Pin, double* __restrict__ Pout, int store,
             unsigned long long* __restrict__ near) {
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const int i = (int)(e / D), c = (int)(e - (long long)i * D);
    double acc = 0.0, mag = 0.0;
    for (int k = row_ptr[i]; k < row_ptr[i + 1]; ++k) {
      const double t = tval[k], p = Pin[(long long)col_idx[k] * D + c];
      acc = fma(t, p, acc);
      mag += fabs(t * p);
    }
    double out = acc;
    bool edge = false;
    if (store == PK_STORE_F32) {
      const float f = (float)acc;
      out = (double)f;
      // the float32 rounding flips where acc is half a float32 ulp away from out
      const float fa = fabsf(f);
      const double ulp = (double)nextafterf(fa, INFINITY) - (double)fa;
      edge = isfinite(acc) && fabs(fabs(acc - out) - 0.5 * ulp) <= PK_MARGIN * fmax(mag, 1e-300);
    } else if (store == PK_STORE_INT) {
      out = trunc(acc);
      edge = acc != 0.0 && pk_near_int(acc, mag);
    }
    if (edge) atomicAdd(near, 1ULL);
    Pout[e] = out;
  }
}

// Which rows of a transform with labels unseen at fit hash with the extended u (propagation.py:328-395): at level 0
// the vertices with a new label, after every propagation the rows whose new-label columns are all positive.  Only the
// transformed graphs' vertices (v >= v0) take part.
__global__ void __launch_bounds__(256)
pk_private(int V, int v0, int D, int dim_orig, int level, const int* __restrict__ labels, const double* __restrict__ P,
           unsigned char* __restrict__ priv) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  bool p = false;
  if (v >= v0) {
    if (level == 0) {
      p = labels[v] >= dim_orig;
    } else {
      p = true;
      for (int c = dim_orig; c < D && p; ++c) p = P[(long long)v * D + c] > 0.0;
    }
  }
  priv[v] = p ? 1 : 0;
}

struct PkHashParams {
  int V, D;
  int attr;               // 1: the d-tuple floor((P_vj u_j + b_j) / w); 0: floor((dot(P_v, u) + b) / w)
  int take_sqrt;          // labelled, M = "H": sqrt(P) first
  int dim_orig;           // labelled: vertices that are not private use columns [0, dim_orig)
  const double* P;
  const double* u;        // [D] of this level
  const double* b;        // [1] or [D] of this level
  double w;
  const unsigned char* priv;  // NULL = no private vertices
  double* bins;           // [V * K] of this level, K = attr ? D : 1; -0.0 stored as +0.0
  unsigned long long* near;
  unsigned* nan_seen;
};

__device__ __forceinline__ double pk_bin(double x, double mag, const PkHashParams& p, int* near, bool* nan) {
  const double f = floor(x);
  if (isnan(f)) *nan = true;
  if (isfinite(x) && pk_near_int(x, mag)) ++*near;
  return f == 0.0 ? 0.0 : f;  // np.unique and dict lookup treat -0.0 and 0.0 as one value
}

// One thread per vertex: the row is read in order from L1 (a fixed-order sum cannot be split across lanes).
__global__ void __launch_bounds__(256)
pk_hash(PkHashParams p) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= p.V) return;
  const double* row = p.P + (long long)v * p.D;
  int near = 0;
  bool nan = false;
  if (p.attr) {
    for (int j = 0; j < p.D; ++j) {
      const double t = __dmul_rn(row[j], p.u[j]);
      const double x = __ddiv_rn(__dadd_rn(t, p.b[j]), p.w);
      p.bins[(long long)v * p.D + j] = pk_bin(x, (fabs(t) + fabs(p.b[j])) / fabs(p.w), p, &near, &nan);
    }
  } else {
    const int n = (p.priv && p.priv[v]) ? p.D : p.dim_orig;
    double acc = 0.0, mag = 0.0;
    for (int c = 0; c < n; ++c) {
      const double x = p.take_sqrt ? sqrt(row[c]) : row[c];
      acc = fma(x, p.u[c], acc);
      mag += fabs(x * p.u[c]);
    }
    const double x = __ddiv_rn(__dadd_rn(acc, p.b[0]), p.w);
    p.bins[v] = pk_bin(x, (mag + fabs(p.b[0])) / fabs(p.w), p, &near, &nan);
  }
  if (near) atomicAdd(p.near, (unsigned long long)near);
  if (nan) atomicOr(p.nan_seen, 1u);
}

// ---- per-level columns: a bin is the K-tuple of the vertex's floors plus its private flag.  A 64-bit fingerprint
// picks the slot; a slot holds the vertex that claimed it, and equality is checked against that vertex's full tuple
// (nh_code_insert with a tuple compare).  nh_code_number then numbers the claimed slots.
__device__ __forceinline__ unsigned long long pk_fingerprint(const double* bins, int K, int v, unsigned char priv) {
  unsigned long long h = priv ? 0x9E3779B97F4A7C15ULL : 0ULL;
  for (int j = 0; j < K; ++j) h = mix64(h ^ (unsigned long long)__double_as_longlong(bins[(long long)v * K + j]));
  return h;
}

__device__ __forceinline__ bool pk_same(const double* bins, const unsigned char* priv, int K, int a, int b) {
  if (priv && priv[a] != priv[b]) return false;
  for (int j = 0; j < K; ++j)
    if (__double_as_longlong(bins[(long long)a * K + j]) != __double_as_longlong(bins[(long long)b * K + j])) return false;
  return true;
}

__global__ void __launch_bounds__(256)
pk_code_insert(int V, int K, const double* __restrict__ bins, const unsigned char* __restrict__ priv,
               int* __restrict__ tab, unsigned mask, int* __restrict__ slot_of) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  unsigned s = (unsigned)pk_fingerprint(bins, K, v, priv ? priv[v] : 0) & mask;
  for (;;) {
    int cur = tab[s];
    if (cur < 0) {
      cur = atomicCAS(&tab[s], -1, v);
      if (cur < 0) break;
    }
    if (pk_same(bins, priv, K, cur, v)) break;
    s = (s + 1) & mask;
  }
  slot_of[v] = (int)s;
}

// (graph, column) counts of one level into the feature table, with the self-similarity / max-count / entry
// bookkeeping of wl_insert_level0.  `extra`: the reference's transform with new labels counts vertex v in every
// transformed graph k with graph_ptr[k] <= v <= graph_ptr[k + 1] (propagation.py:371-383), so the first vertex of a
// graph also counts in the graph before it (and across empty graphs); those counts go to partial slots of their own.
__global__ void __launch_bounds__(256)
pk_count(int V, const int* __restrict__ vgraph, const int* __restrict__ graph_ptr, const int* __restrict__ slot_of,
         const int* __restrict__ colid, unsigned long long* ft_keys, unsigned* ft_cnt, unsigned ft_mask, FeatStats st,
         int level, int extra, int g_y0, size_t extra_part) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  bool did = false, is_new = false;
  int g = 0;
  unsigned old = 0, col = 0;
  if (v < V) {
    g = vgraph[v];
    col = (unsigned)colid[slot_of[v]];
    old = ft_add(ft_keys, ft_cnt, ft_mask, ((unsigned long long)(unsigned)g << 32) | col, 1u, st, &is_new);
    did = true;
  }
  ft_account(did, g, old, is_new, st, (size_t)level * gridDim.x + blockIdx.x);
  if (!extra || !did) return;
  for (int k = g - 1; k >= g_y0 && graph_ptr[k + 1] == v; --k) {
    bool nw;
    const unsigned o = ft_add(ft_keys, ft_cnt, ft_mask, ((unsigned long long)(unsigned)k << 32) | col, 1u, st, &nw);
    atomicAdd(&st.diag[k], 2ULL * o + 1ULL);
    atomicMax(&st.part_max[extra_part + blockIdx.x], o + 1);
    if (nw) atomicAdd(&st.part_new[extra_part + blockIdx.x], 1u);
  }
}

}  // namespace gk
