// GraphHopper kernel (reference: graph_hopper.py:19-449, Feragen et al. 2013).
//
// For every root j the reference builds a DAG on the vertices j reaches (unit weights):
//   u -> v  if u is v's Dijkstra predecessor -- the smallest-id in-neighbour with D_j(u) = D_j(v) - 1 -- unless u
//           is the smallest vertex id reachable from j (the `p_cc[v] > 0` test on the compacted index, :213);
//   u -> v  for every OUT-neighbour u of v with D_j(u) = D_j(v) - 1 (:221-231).
// sigma_j(v) counts DAG paths j ~> v, des_j(v, l) DAG paths of length l leaving v (od_vectors_dag, :386-449), and
//   M[v, a, b] = sum_j [a = D_j(v)] sigma_j(v) des_j(v, b - a)        (a <= b < delta, :250-260)
// is kept as its upper triangle: row v holds T = delta (delta + 1) / 2 doubles, (a, b) at a delta - a (a - 1) / 2 + b - a.
// The pair kernel is sum_{v in G, v' in G'} <M_v, M_v'> k(x_v, x_v') (:268-365).
#pragma once
#include "common.cuh"

namespace gk {

constexpr int GH_THREADS = 128;
constexpr int GH_GROUP_NODES = 128;  // node-pair Gram: vertices of one graph group (a larger graph is a group alone)
constexpr int GH_GROUP_GRAPHS = 32;  // ... and graphs of one group
constexpr int GH_TILE = 64;          // node sub-tile of the node-pair Gram
enum { GH_NK_LINEAR = 0, GH_NK_GAUSSIAN = 1, GH_NK_BRIDGE = 2 };

struct GhParams {
  const int* graph_ptr;
  const int* row_ptr;
  const int* col_idx;
  const int* glist;        // graphs of this launch
  unsigned char* ws;       // global workspace (graphs whose working set does not fit shared memory)
  const long long* woff;   // byte offset of each graph's workspace in ws
  int ws_global;
  int* gdiam;              // [N] largest eccentricity of each graph (written by the first pass)
  int* delta_max;          // max over graphs of gdiam + 1
  double* M;               // [V][T]
  int delta;
  long long T;
};

// Working set of one graph: MAPS = false (eccentricities) needs the BFS arrays only.
__host__ __device__ inline size_t gh_ws_bytes(long long n, int dg, bool maps) {
  const size_t ints = (size_t)(4 * n + 2) * 4;
  const size_t longs = maps ? (size_t)n * (1 + dg) * 8 : 0;
  return (longs + ints + 15) / 16 * 16;
}

// One CTA per graph, roots in ascending order.  Per root: level-synchronous BFS over the CSR (distances, BFS order,
// level offsets, the min-id predecessor by integer atomicMin), then sigma forward and des backward over the DAG
// (integer sums: the result does not depend on the order inside a level), then M += sigma * des, each vertex's row
// written by one thread -- M is deterministic and exact while its entries stay below 2^53.
template <bool MAPS>
__global__ void __launch_bounds__(GH_THREADS)
gh_dag_kernel(GhParams p) {
  extern __shared__ __align__(16) unsigned char gh_smem[];
  const int g = p.glist[blockIdx.x];
  const int v0 = p.graph_ptr[g];
  const int n = p.graph_ptr[g + 1] - v0;
  const int tid = threadIdx.x;
  if (n <= 0) {
    if (!MAPS && tid == 0) p.gdiam[g] = 0;
    return;
  }
  unsigned char* base = p.ws_global ? p.ws + p.woff[g] : gh_smem;
  const int dg = MAPS ? p.gdiam[g] + 1 : 0;  // row length of des
  long long* sigma = reinterpret_cast<long long*>(base);  // [n]
  long long* des = sigma + n;                              // [n][dg]
  int* dist = reinterpret_cast<int*>(MAPS ? (unsigned char*)(des + (size_t)n * dg) : base);  // [n], -1 = unreached
  int* order = dist + n;                                   // [n] BFS order, levels contiguous
  int* lvl = order + n;                                    // [n + 2] level offsets into order
  int* pred = lvl + n + 2;                                 // [n] smallest-id in-neighbour one level up
  const int* rp = p.row_ptr + v0;
  __shared__ int s_cnt, s_minr, s_ecc;
  if (tid == 0) s_ecc = 0;
  for (int root = 0; root < n; ++root) {
    for (int i = tid; i < n; i += GH_THREADS) { dist[i] = -1; pred[i] = 0x7fffffff; }
    __syncthreads();
    if (tid == 0) { dist[root] = 0; order[0] = root; lvl[0] = 0; lvl[1] = 1; s_cnt = 1; s_minr = root; }
    __syncthreads();
    int L = 0;
    while (true) {
      const int b = lvl[L], e = lvl[L + 1];
      if (b == e) break;  // uniform: lvl is read after a barrier
      for (int i = b + tid; i < e; i += GH_THREADS) {
        const int u = order[i];
        for (int k = rp[u]; k < rp[u + 1]; ++k) {
          const int w = p.col_idx[k] - v0;
          if (w == u) continue;  // self-loops take no part (graph_hopper.py:183)
          const int old = atomicCAS(&dist[w], -1, L + 1);
          if (old == -1) {
            order[atomicAdd(&s_cnt, 1)] = w;
            atomicMin(&s_minr, w);
          }
          if (MAPS && (old == -1 || old == L + 1)) atomicMin(&pred[w], u);
        }
      }
      __syncthreads();
      if (tid == 0) lvl[L + 2] = s_cnt;
      __syncthreads();
      ++L;
    }
    const int ecc = L - 1;
    if (!MAPS) {
      if (tid == 0) s_ecc = max(s_ecc, ecc);
      continue;
    }
    const int nr = s_cnt, minr = s_minr;
    // sigma, level by level: the DAG parents of v are its out-neighbours one level up, plus pred(v) unless it is the
    // smallest reachable id
    if (tid == 0) sigma[root] = 1;
    __syncthreads();
    for (int l = 1; l <= ecc; ++l) {
      for (int i = lvl[l] + tid; i < lvl[l + 1]; i += GH_THREADS) {
        const int v = order[i], pv = pred[v];
        long long s = 0;
        bool seen = false;
        for (int k = rp[v]; k < rp[v + 1]; ++k) {
          const int u = p.col_idx[k] - v0;
          if (u != v && dist[u] == l - 1) { s += sigma[u]; seen |= u == pv; }
        }
        if (!seen && pv != minr) s += sigma[pv];
        sigma[v] = s;
      }
      __syncthreads();
    }
    // des: des(v, 0) = 1, pushed to the parents from the deepest level up (integer atomics)
    for (int i = tid; i < nr; i += GH_THREADS) {
      const int v = order[i];
      long long* dv = des + (size_t)v * dg;
      dv[0] = 1;
      for (int l = 1; l <= ecc - dist[v]; ++l) dv[l] = 0;
    }
    __syncthreads();
    for (int l = ecc; l >= 1; --l) {
      for (int i = lvl[l] + tid; i < lvl[l + 1]; i += GH_THREADS) {
        const int v = order[i], pv = pred[v];
        const long long* dv = des + (size_t)v * dg;
        const int len = ecc - l + 1;
        bool seen = false;
        for (int k = rp[v]; k < rp[v + 1]; ++k) {
          const int u = p.col_idx[k] - v0;
          if (u != v && dist[u] == l - 1) {
            seen |= u == pv;
            unsigned long long* du = reinterpret_cast<unsigned long long*>(des + (size_t)u * dg);
            for (int t = 0; t < len; ++t) atomicAdd(du + t + 1, (unsigned long long)dv[t]);
          }
        }
        if (!seen && pv != minr) {
          unsigned long long* du = reinterpret_cast<unsigned long long*>(des + (size_t)pv * dg);
          for (int t = 0; t < len; ++t) atomicAdd(du + t + 1, (unsigned long long)dv[t]);
        }
      }
      __syncthreads();
    }
    for (int i = tid; i < nr; i += GH_THREADS) {
      const int v = order[i], a = dist[v];
      double* row = p.M + (size_t)(v0 + v) * p.T + ((long long)a * p.delta - (long long)a * (a - 1) / 2);
      const long long* dv = des + (size_t)v * dg;
      const long long sv = sigma[v];
      for (int l = 0; l <= ecc - a; ++l) row[l] += (double)(sv * dv[l]);
    }
    __syncthreads();
  }
  if (!MAPS && tid == 0) {
    p.gdiam[g] = s_ecc;
    atomicMax(p.delta_max, s_ecc + 1);
  }
}

// Linear node kernel: Phi[g][t * d + k] = sum_{v in g} M[v][t] x_v[k] (vertices in ascending order).
__global__ void __launch_bounds__(256)
gh_linear_features(const int* __restrict__ graph_ptr, const double* __restrict__ M, long long T,
                   const double* __restrict__ attrs, int d, double* __restrict__ phi) {
  const int g = blockIdx.x;
  const int v0 = graph_ptr[g], v1 = graph_ptr[g + 1];
  const long long D = T * d;
  for (long long e = threadIdx.x; e < D; e += 256) {
    const long long t = e / d;
    const int k = (int)(e - t * d);
    double s = 0.0;
    for (int v = v0; v < v1; ++v) s = fma(M[(size_t)v * T + t], attrs[(size_t)v * d + k], s);
    phi[(size_t)g * D + e] = s;
  }
}

template <int NK>
__device__ __forceinline__ double gh_node_kernel(double sqdist, double mu) {
  if constexpr (NK == GH_NK_GAUSSIAN) return exp(-mu * sqdist);
  else return fmax(0.0, (4.0 - sqrt(sqdist)) * 0.25);
}

// Self similarity of every graph for the node-pair kernels: one CTA per graph, node pairs strided over the threads,
// partials summed in a fixed order (no floating-point atomics).
template <int NK>
__global__ void __launch_bounds__(256)
gh_nodepair_diag(const int* __restrict__ graph_ptr, const double* __restrict__ M, long long T,
                 const double* __restrict__ attrs, int d, double mu, double* __restrict__ diag) {
  const int g = blockIdx.x;
  const int v0 = graph_ptr[g], n = graph_ptr[g + 1] - v0;
  __shared__ double red[8];
  double s = 0.0;
  for (long long q = threadIdx.x; q < (long long)n * n; q += 256) {
    const int a = v0 + (int)(q / n), b = v0 + (int)(q % n);
    const double* ma = M + (size_t)a * T;
    const double* mb = M + (size_t)b * T;
    double w = 0.0, sq = 0.0;
    for (long long t = 0; t < T; ++t) w = fma(ma[t], mb[t], w);
    for (int k = 0; k < d; ++k) {
      const double df = attrs[(size_t)a * d + k] - attrs[(size_t)b * d + k];
      sq = fma(df, df, sq);
    }
    s += w * gh_node_kernel<NK>(sq, mu);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < 8; ++w) t += red[w];
    diag[g] = t;
  }
}

struct GhGramParams {
  const int* graph_ptr;
  const double* M;
  long long T;
  const double* attrs;
  int d;
  double mu;
  const int2* pairs;     // (row group, column group) of each CTA
  const int* rgroups;    // first graph of each row group (+ end)
  const int* cgroups;    // first graph of each column group (+ end)
  int square;            // symmetric case: upper entries only, mirrored
  int a0, a1;            // rows of K that are written (graph indices)
  int row0;              // graph index of output row 0
  double* out;
  long long ld;
};

// Node-pair Gram of two graph groups: for every 64 x 64 node sub-tile, P[v][v'] = <M_v, M_v'> k(x_v, x_v') in fp64
// CUDA-core FMAs (16 x 16 threads, 4 x 4 each; ||x_v - x_v'||^2 summed directly), then a fixed-order segmented
// reduction: each row's columns per column graph, then those per row graph, into the group pair's accumulators.
// Deterministic (no floating-point atomics); in the symmetric case a CTA (I, J) with I <= J writes the entries
// (g, g') with g < g' and their mirror, so K is exactly symmetric and a row block equals the same rows of the full K.
template <int NK>
__global__ void __launch_bounds__(256)
gh_nodepair_gram(GhGramParams p) {
  extern __shared__ __align__(16) unsigned char gh_smem[];
  double* As = reinterpret_cast<double*>(gh_smem);          // [16][65]
  double* Bs = As + 16 * 65;                                 // [16][65]
  double* Ps = Bs + 16 * 65;                                 // [64][65]
  double* Rs = Ps + GH_TILE * 65;                            // [64][GH_GROUP_GRAPHS]
  double* acc = Rs + GH_TILE * GH_GROUP_GRAPHS;              // [GH_GROUP_GRAPHS][GH_GROUP_GRAPHS]
  __shared__ int rgp[GH_GROUP_GRAPHS + 1], cgp[GH_GROUP_GRAPHS + 1];
  const int2 pr = p.pairs[blockIdx.x];
  const int rg0 = p.rgroups[pr.x], rg1 = p.rgroups[pr.x + 1];
  const int cg0 = p.cgroups[pr.y], cg1 = p.cgroups[pr.y + 1];
  const int nI = rg1 - rg0, nJ = cg1 - cg0;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  for (int i = tid; i <= nI; i += 256) rgp[i] = p.graph_ptr[rg0 + i];
  for (int i = tid; i <= nJ; i += 256) cgp[i] = p.graph_ptr[cg0 + i];
  for (int i = tid; i < nI * nJ; i += 256) acc[i] = 0.0;
  __syncthreads();
  const int rv0 = rgp[0], rv1 = rgp[nI], cv0 = cgp[0], cv1 = cgp[nJ];
  const long long T = p.T;
  const int d = p.d;
  for (int rs = rv0; rs < rv1; rs += GH_TILE) {
    const int re = min(rv1, rs + GH_TILE);
    for (int cs = cv0; cs < cv1; cs += GH_TILE) {
      const int ce = min(cv1, cs + GH_TILE);
      double w[4][4] = {}, sq[4][4] = {};
      for (long long k0 = 0; k0 < T; k0 += 16) {
        for (int i = tid; i < GH_TILE * 16; i += 256) {
          const int r = i >> 4, k = i & 15;
          const long long kk = k0 + k;
          As[k * 65 + r] = (rs + r < re && kk < T) ? p.M[(size_t)(rs + r) * T + kk] : 0.0;
          Bs[k * 65 + r] = (cs + r < ce && kk < T) ? p.M[(size_t)(cs + r) * T + kk] : 0.0;
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < 16; ++k) {
          double a[4], b[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) { a[i] = As[k * 65 + ty * 4 + i]; b[i] = Bs[k * 65 + tx * 4 + i]; }
#pragma unroll
          for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) w[i][j] = fma(a[i], b[j], w[i][j]);
        }
        __syncthreads();
      }
      for (int k0 = 0; k0 < d; k0 += 16) {
        for (int i = tid; i < GH_TILE * 16; i += 256) {
          const int r = i >> 4, k = i & 15;
          const int kk = k0 + k;
          As[k * 65 + r] = (rs + r < re && kk < d) ? p.attrs[(size_t)(rs + r) * d + kk] : 0.0;
          Bs[k * 65 + r] = (cs + r < ce && kk < d) ? p.attrs[(size_t)(cs + r) * d + kk] : 0.0;
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < 16; ++k) {
          double a[4], b[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) { a[i] = As[k * 65 + ty * 4 + i]; b[i] = Bs[k * 65 + tx * 4 + i]; }
#pragma unroll
          for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const double df = a[i] - b[j];
              sq[i][j] = fma(df, df, sq[i][j]);
            }
        }
        __syncthreads();
      }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
          Ps[(ty * 4 + i) * 65 + tx * 4 + j] = w[i][j] * gh_node_kernel<NK>(sq[i][j], p.mu);
      __syncthreads();
      // rows: sum of each row's columns inside every column graph
      for (int e = tid; e < (re - rs) * nJ; e += 256) {
        const int r = e / nJ, gj = e - r * nJ;
        const int c0 = max(cgp[gj], cs), c1 = min(cgp[gj + 1], ce);
        double s = 0.0;
        for (int c = c0; c < c1; ++c) s += Ps[r * 65 + (c - cs)];
        Rs[r * GH_GROUP_GRAPHS + gj] = s;
      }
      __syncthreads();
      for (int e = tid; e < nI * nJ; e += 256) {
        const int gi = e / nJ, gj = e - gi * nJ;
        const int r0 = max(rgp[gi], rs), r1 = min(rgp[gi + 1], re);
        if (r0 >= r1 || max(cgp[gj], cs) >= min(cgp[gj + 1], ce)) continue;
        double s = 0.0;
        for (int r = r0; r < r1; ++r) s += Rs[(r - rs) * GH_GROUP_GRAPHS + gj];
        acc[e] += s;
      }
      __syncthreads();
    }
  }
  for (int e = tid; e < nI * nJ; e += 256) {
    const int gi = e / nJ, gj = e - gi * nJ;
    const int g = rg0 + gi, h = cg0 + gj;
    if (p.square) {
      if (g >= h) continue;
      if (g >= p.a0 && g < p.a1) p.out[(long long)(g - p.row0) * p.ld + h] = acc[e];
      if (h >= p.a0 && h < p.a1) p.out[(long long)(h - p.row0) * p.ld + g] = acc[e];
    } else if (g >= p.a0 && g < p.a1) {
      p.out[(long long)(g - p.row0) * p.ld + h] = acc[e];
    }
  }
}

constexpr size_t GH_GRAM_SMEM = (size_t)(2 * 16 * 65 + GH_TILE * 65 + GH_TILE * GH_GROUP_GRAPHS +
                                         GH_GROUP_GRAPHS * GH_GROUP_GRAPHS) * 8;

}  // namespace gk
