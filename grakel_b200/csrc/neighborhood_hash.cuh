// NeighborhoodHash (Hido & Kashima 2009; neighborhood_hash.py:14-570) on the device.
//
// Every level relabels each vertex with a bit rotation of its own code XOR-ed with its out-neighbours' codes
// (simple) or with one rotated term per run of radix_sort_rot (count sensitive, below).  Codes
// are u64: the reference's Python ints never leave that range (a masked rotation is < 2^bits <= 2^64, a count is
// < 2^31).  A vertex whose own code or any neighbour's code is None stays None (transform: labels unseen at fit).
//
// The pair value of level r is the multiset intersection c_r = sum_code min(cnt_i, cnt_j) of the two graphs'
// non-None codes, i.e. the WL-OA histogram intersection: every level's codes are compacted into dense column ids,
// counted per graph, unary-expanded (wl_oa.cuh) and fed to the exact integer Gram of gk_gram, one level at a
// time (the combine below is not linear in c, so levels never share columns).  nh_combine then evaluates the
// reference's fp64 expression  sum(t_r) / R,  t_r = c_r / (n_i + n_j - c_r),  with CPython's float `sum`.
#pragma once
#include "common.cuh"
#include "wl.cuh"

namespace gk {

// ROT(n, d) of neighborhood_hash.py:367-390.  m = d % bits; 0 < m < bits <= 64 keeps both shifts defined.
__device__ __forceinline__ unsigned long long nh_rot(unsigned long long n, unsigned long long d, int bits,
                                                     unsigned long long mask) {
  const int m = (int)(d % (unsigned long long)bits);
  if (m == 0) return n;
  return ((n << m) & mask) | ((n & mask) >> (bits - m));
}

// level-0 input: code and None flag of every vertex from its dense label id
__global__ void __launch_bounds__(256)
nh_init(int V, const int* __restrict__ labels, const unsigned long long* __restrict__ code_of_label,
        const unsigned char* __restrict__ label_valid, unsigned long long* __restrict__ codes,
        unsigned char* __restrict__ valid) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  const int l = labels[v];
  codes[v] = code_of_label[l];
  valid[v] = label_valid[l];
}

constexpr int NH_SIMPLE = 0, NH_COUNT = 1;

// Count sensitive (radix_sort_rot, neighborhood_hash.py:449-504): the neighbour codes, in the order of the edge
// dictionary, are sorted STABLY by their low `bits` bits only (an LSD radix sort), and every maximal run of equal
// consecutive values contributes ROT(value ^ run, run).  From level 1 on a code can exceed the mask (ROT(x, d) is x
// unmasked when d % bits == 0), so two different codes can share a sort key; they then stay interleaved in
// neighbour order and form separate runs.  Runs never span two keys, so the result is the XOR over the keys of the
// runs of each key's subsequence in neighbour order -- no sort needed.  A key holding two different codes makes the
// result depend on the neighbour order: such vertices raise *order_dep (the caller may not know the reference's order).

// One thread per vertex of degree <= width (the rest are in the large list).  Count sensitive: position i starts a
// run unless the nearest earlier neighbour with its key holds the same code; the run goes on over the later
// neighbours with that key while they hold the same code -- O(deg^2) loads of L1-resident codes for deg <= 32.
template <int MODE>
__global__ void __launch_bounds__(256)
nh_hash_small(int V, int width, const int* __restrict__ row_ptr, const int* __restrict__ col_idx,
              const unsigned long long* __restrict__ in, const unsigned char* __restrict__ vin,
              unsigned long long* __restrict__ out, unsigned char* __restrict__ vout, int bits, unsigned long long mask,
              unsigned* __restrict__ order_dep) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  const int b = row_ptr[v], e = row_ptr[v + 1];
  if (e - b > width) return;
  bool ok = vin[v] != 0;
  for (int i = b; i < e && ok; ++i) ok = vin[col_idx[i]] != 0;
  if (!ok) {
    out[v] = 0ULL;
    vout[v] = 0;
    return;
  }
  unsigned long long acc = 0ULL;
  if (MODE == NH_SIMPLE) {
    for (int i = b; i < e; ++i) acc ^= in[col_idx[i]];
  } else {
    bool mixed = false;
    for (int i = b; i < e; ++i) {
      const unsigned long long c = in[col_idx[i]], k = c & mask;
      bool start = true;
      for (int j = i - 1; j >= b; --j) {
        const unsigned long long cj = in[col_idx[j]];
        if ((cj & mask) == k) { start = cj != c; break; }
      }
      if (!start) continue;
      unsigned long long occ = 1;
      for (int j = i + 1; j < e; ++j) {
        const unsigned long long cj = in[col_idx[j]];
        if ((cj & mask) != k) continue;
        if (cj != c) { mixed = true; break; }
        ++occ;
      }
      acc ^= nh_rot(c ^ occ, occ, bits, mask);
    }
    if (mixed) atomicOr(order_dep, 1u);
  }
  out[v] = nh_rot(in[v], 1ULL, bits, mask) ^ acc;
  vout[v] = 1;
}

constexpr int NH_LARGE_THREADS = 256;

// One CTA per vertex of the large list (degree > width).  Count sensitive: the sort keys go through an
// open-addressing table of 2 deg slots at [2 row_ptr[v], 2 row_ptr[v+1]) of a global workspace; a slot holds the row
// position of one neighbour with its key (codes span all 2^64 values, so no code can mark a free slot), the key's
// neighbour count and whether the key holds two different codes.  A key with one code is one run of that count.  The
// keys with two or more codes (rare: they need counts that are multiples of bits) are walked by one thread in
// neighbour order, a slot then holding its current run (start position, length).  Any degree works, e.g. a star with
// more leaves than 2^bits.
template <int MODE>
__global__ void __launch_bounds__(NH_LARGE_THREADS)
nh_hash_large(const int* __restrict__ large_list, const int* __restrict__ row_ptr, const int* __restrict__ col_idx,
              const unsigned long long* __restrict__ in, const unsigned char* __restrict__ vin,
              unsigned long long* __restrict__ out, unsigned char* __restrict__ vout, int bits, unsigned long long mask,
              int* __restrict__ tab, unsigned* __restrict__ tcnt, unsigned* __restrict__ order_dep) {
  __shared__ unsigned long long s_x[NH_LARGE_THREADS / 32];
  const int v = large_list[blockIdx.x];
  const int b = row_ptr[v], e = row_ptr[v + 1];
  int ok = 1;
  for (int i = b + threadIdx.x; i < e; i += NH_LARGE_THREADS) ok &= vin[col_idx[i]] != 0;
  ok = __syncthreads_and(ok) && vin[v] != 0;
  if (!ok) {
    if (threadIdx.x == 0) { out[v] = 0ULL; vout[v] = 0; }
    return;
  }
  unsigned long long acc = 0ULL;
  if (MODE == NH_SIMPLE) {
    for (int i = b + threadIdx.x; i < e; i += NH_LARGE_THREADS) acc ^= in[col_idx[i]];
  } else {
    const long long S = 2LL * (e - b);
    int* t = tab + 2LL * b;
    unsigned* tc = tcnt + 4LL * b;  // [2 deg] counts | [2 deg] "two codes" flags
    unsigned* tm = tc + S;
    for (long long s = threadIdx.x; s < S; s += NH_LARGE_THREADS) { t[s] = -1; tc[s] = 0u; tm[s] = 0u; }
    __syncthreads();
    for (int i = b + threadIdx.x; i < e; i += NH_LARGE_THREADS) {
      const unsigned long long c = in[col_idx[i]], k = c & mask;
      long long s = (long long)(mix64(k) % (unsigned long long)S);
      for (;;) {
        int cur = t[s];
        if (cur < 0) {
          cur = atomicCAS(&t[s], -1, i);
          if (cur < 0) { atomicAdd(&tc[s], 1u); break; }
        }
        const unsigned long long cc = in[col_idx[cur]];
        if ((cc & mask) == k) {
          atomicAdd(&tc[s], 1u);
          if (cc != c) tm[s] = 1u;
          break;
        }
        s = s + 1 == S ? 0 : s + 1;
      }
    }
    __syncthreads();
    int mixed = 0;
    for (long long s = threadIdx.x; s < S; s += NH_LARGE_THREADS) {
      const int r = t[s];
      if (r < 0) continue;
      if (tm[s]) { mixed = 1; tc[s] = 0u; continue; }
      const unsigned long long c = in[col_idx[r]], occ = tc[s];
      acc ^= nh_rot(c ^ occ, occ, bits, mask);
    }
    if (__syncthreads_or(mixed) && threadIdx.x == 0) {
      atomicOr(order_dep, 1u);
      for (int i = b; i < e; ++i) {  // the keys with several codes, in neighbour order
        const unsigned long long c = in[col_idx[i]], k = c & mask;
        long long s = (long long)(mix64(k) % (unsigned long long)S);
        while ((in[col_idx[t[s]]] & mask) != k) s = s + 1 == S ? 0 : s + 1;
        if (!tm[s]) continue;
        if (tc[s] && in[col_idx[t[s]]] == c) { ++tc[s]; continue; }
        if (tc[s]) acc ^= nh_rot(in[col_idx[t[s]]] ^ tc[s], tc[s], bits, mask);
        t[s] = i;
        tc[s] = 1u;
      }
      for (long long s = 0; s < S; ++s)
        if (t[s] >= 0 && tm[s] && tc[s]) acc ^= nh_rot(in[col_idx[t[s]]] ^ tc[s], tc[s], bits, mask);
    }
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) acc ^= __shfl_xor_sync(0xffffffffu, acc, d);
  if ((threadIdx.x & 31) == 0) s_x[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < NH_LARGE_THREADS / 32; ++w) acc ^= s_x[w];
    out[v] = nh_rot(in[v], 1ULL, bits, mask) ^ acc;
    vout[v] = 1;
  }
}

// ---- per-level columns: distinct codes -> dense ids (any order: K does not depend on the column numbering)
// pass 1: every non-None vertex finds (or claims) the slot of its code; a slot holds its claimer's vertex id
__global__ void __launch_bounds__(256)
nh_code_insert(int V, const unsigned long long* __restrict__ codes, const unsigned char* __restrict__ valid,
               int* __restrict__ tab, unsigned mask, int* __restrict__ slot_of) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V || !valid[v]) return;
  const unsigned long long c = codes[v];
  unsigned s = (unsigned)mix64(c) & mask;
  for (;;) {
    int cur = tab[s];
    if (cur < 0) {
      cur = atomicCAS(&tab[s], -1, v);
      if (cur < 0) break;
    }
    if (codes[cur] == c) break;
    s = (s + 1) & mask;
  }
  slot_of[v] = (int)s;
}

// pass 2: the claimer of a slot numbers its column
__global__ void __launch_bounds__(256)
nh_code_number(int V, const unsigned char* __restrict__ valid, const int* __restrict__ tab,
               const int* __restrict__ slot_of, int* __restrict__ colid, unsigned long long* n_cols) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V || !valid[v]) return;
  const int s = slot_of[v];
  if (tab[s] == v) colid[s] = (int)atomicAdd(n_cols, 1ULL);
}

// pass 3: (graph, column) -> count, the (graph << 32 | column) element layout of the SP / WL feature tables.
// Entry v belongs to vertex v / per (NeighborhoodHash: one entry per vertex; PyramidMatch: d per vertex).
__global__ void __launch_bounds__(256)
nh_count(int V, int per, const unsigned char* __restrict__ valid, const int* __restrict__ vgraph,
         const int* __restrict__ slot_of, const int* __restrict__ colid, unsigned long long* __restrict__ keys,
         unsigned* __restrict__ cnt, unsigned mask) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V || !valid[v]) return;
  const unsigned long long key = ((unsigned long long)(unsigned)vgraph[v / per] << 32) | (unsigned)colid[slot_of[v]];
  unsigned s = (unsigned)mix64(key) & mask;
  for (;;) {
    unsigned long long cur = keys[s];
    if (cur == EMPTY64) {
      cur = atomicCAS(&keys[s], EMPTY64, key);
      if (cur == EMPTY64) cur = key;
    }
    if (cur == key) { atomicAdd(&cnt[s], 1u); return; }
    s = (s + 1) & mask;
  }
}

// ---- combine: K = sum(t_r) / R, t_r = c_r / (n_i + n_j - c_r), as the reference evaluates it
// (neighborhood_hash.py:340-341, 570).  c_r are exact integers in fp32 (every entry <= min(n_i, n_j) < 2^26), the
// graph sizes are exact; each division and addition is one correctly rounded IEEE operation (no contraction, no
// reciprocal).  A 32 x 32 tile per CTA; `mirror` (full square matrix): only tiles with tj >= ti run and the
// transposed tile is written through shared memory, so K is exactly symmetric and the counts are read once.
constexpr int NH_TILE = 32;

struct NhCombineParams {
  const float* C;         // R matrices [rows x ldc], level r at C + r * stride
  long long stride, ldc;
  int R;
  const int* graph_ptr;
  int row_g0;             // graph of row 0
  int rows, cols;         // the block's rows (graphs row_g0 + i) and columns (graphs j)
  int mirror;
  double* out;
  long long ld;
};

// The sum is CPython's built-in `sum` of floats (Python >= 3.12): 0 + t_0 is exact, every later term goes through
// Neumaier's compensated addition, and the compensation is added once at the end when it is non-zero and finite.
__device__ __forceinline__ double nh_value(const NhCombineParams& p, int i, int j, int ni, int nj) {
  const double nn = (double)(ni + nj);
  const long long off = (long long)i * p.ldc + j;
  // IEEE round-to-nearest division (nvcc's default -prec-div=true) and additions; nothing here multiplies, so no
  // contraction into an FMA can change a result
  const double c0 = (double)p.C[off];
  double s = c0 / (nn - c0), comp = 0.0;
  for (int r = 1; r < p.R; ++r) {
    const double c = (double)p.C[(long long)r * p.stride + off];
    const double x = c / (nn - c);
    const double t = s + x;
    comp += fabs(s) >= fabs(x) ? (s - t) + x : (x - t) + s;
    s = t;
  }
  if (comp != 0.0 && isfinite(comp)) s += comp;
  return s / (double)p.R;
}

__global__ void __launch_bounds__(NH_TILE * 8)
nh_combine(NhCombineParams p) {
  __shared__ double s_t[NH_TILE][NH_TILE + 1];
  const int nbj = (p.cols + NH_TILE - 1) / NH_TILE;
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
  const int tx = threadIdx.x & (NH_TILE - 1), ty = threadIdx.x / NH_TILE;
  const int j = tj * NH_TILE + tx;
  const int nj = j < p.cols ? p.graph_ptr[j + 1] - p.graph_ptr[j] : 0;
  for (int k = ty; k < NH_TILE; k += 8) {
    const int i = ti * NH_TILE + k;
    if (i >= p.rows || j >= p.cols) continue;
    const int g = p.row_g0 + i;
    const int ni = p.graph_ptr[g + 1] - p.graph_ptr[g];
    const double x = nh_value(p, i, j, ni, nj);
    p.out[(long long)i * p.ld + j] = x;
    if (p.mirror) s_t[k][tx] = x;
  }
  if (!p.mirror || ti == tj) return;
  __syncthreads();
  // transposed tile: row tj * 32 + k, column ti * 32 + tx  <-  s_t[tx][k]
  for (int k = ty; k < NH_TILE; k += 8) {
    const int r = tj * NH_TILE + k, c = ti * NH_TILE + tx;
    if (r < p.rows && c < p.cols) p.out[(long long)r * p.ld + c] = s_t[tx][k];
  }
}

}  // namespace gk
