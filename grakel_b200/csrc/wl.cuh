// Weisfeiler-Lehman relabelling on the device, all graphs at once.
//
// Replaces weisfeiler_lehman.py:212-258 (generate_graphs: credential =
// own label + sorted out-neighbour labels, global dedup per level) of the
// reference.  The reference dedups exact string credentials; here each vertex
// signature (own label, sorted neighbour-label multiset) is hashed to 64 bits,
// deduplicated in an open-addressing table, and then VERIFIED element by element
// against the representative of its hash slot, so the resulting label partition
// is exact (a detected collision makes the host retry the whole pass with a new
// seed).  New labels are dense ids in first-occurrence (vertex) order.
#pragma once
#include "common.cuh"

namespace gk {

__host__ __device__ __forceinline__ unsigned long long mix64(unsigned long long x) {
  x ^= x >> 33;
  x *= 0xff51afd7ed558ccdULL;
  x ^= x >> 33;
  x *= 0xc4ceb9fe1a85ec53ULL;
  x ^= x >> 33;
  return x;
}

// positional term of the signature hash: value x at sorted position pos
__device__ __forceinline__ unsigned long long sig_term(int x, int pos, unsigned long long seed) {
  return mix64((unsigned long long)(unsigned)x * 0x9E3779B97F4A7C15ULL +
               (unsigned long long)(unsigned)pos * 0xC2B2AE3D27D4EB4FULL + seed);
}

__device__ __forceinline__ unsigned long long sig_final(unsigned long long acc, int own, int deg,
                                                         unsigned long long seed) {
  unsigned long long h = mix64(acc ^ mix64(((unsigned long long)(unsigned)own << 32 | (unsigned)deg) + seed));
  return h >> 1;  // never equals EMPTY64
}

// insert (key -> min vertex id) ; returns the slot.  Popular signatures are hit by
// thousands of vertices: an L2 read (ld.cg) filters out the CAS / atomicMin once the
// key is present / the representative is already smaller, so hot slots do not serialise.
__device__ __forceinline__ unsigned ht_insert(unsigned long long* keys, int* rep, unsigned mask,
                                              unsigned long long key, int v) {
  unsigned slot = (unsigned)(key * 0x9E3779B97F4A7C15ULL >> 20) & mask;
  while (true) {
    unsigned long long prev = __ldcg(&keys[slot]);
    if (prev == EMPTY64) prev = atomicCAS(&keys[slot], EMPTY64, key);
    if (prev == EMPTY64 || prev == key) {
      if (__ldcg(&rep[slot]) > v) atomicMin(&rep[slot], v);
      return slot;
    }
    slot = (slot + 1) & mask;
  }
}

// ---------------------------------------------------------------------------
// K1a: G lanes per vertex, degree <= G.  Coalesced read of the neighbour list,
// label gather (cache-resident: a graph's vertices are contiguous), bitonic sort
// in registers via shuffles, positional 64-bit hash, table insert.
// degen != 0 (tests, gk_selftest_wl_collision): the key leaves the neighbour terms out, so vertices with equal own label
// and degree share a slot and only wl_resolve's verification can separate their classes.
template <int G>
__global__ void __launch_bounds__(256)
wl_sig_small(int V, const int* __restrict__ row_ptr, const int* __restrict__ col_idx,
             const int* __restrict__ lab_in, int* __restrict__ sig_nbr, unsigned long long seed, int degen,
             unsigned long long* ht_keys, int* ht_rep, unsigned ht_mask, int* __restrict__ slot_of) {
  const int tid = blockIdx.x * blockDim.x + threadIdx.x;
  const int v = tid / G;
  const int lane = threadIdx.x & (G - 1);
  int beg = 0, deg = 0;
  bool active = false;
  if (v < V) {
    beg = row_ptr[v];
    deg = row_ptr[v + 1] - beg;
    active = deg <= G;
  }
  int x = 0x7fffffff;
  if (active && lane < deg) x = lab_in[col_idx[beg + lane]];
#pragma unroll
  for (int k = 2; k <= G; k <<= 1) {
#pragma unroll
    for (int j = k >> 1; j > 0; j >>= 1) {
      int y = __shfl_xor_sync(0xffffffffu, x, j);
      bool up = (lane & k) == 0;
      bool lower = (lane & j) == 0;
      x = (lower == up) ? min(x, y) : max(x, y);
    }
  }
  unsigned long long t = 0;
  if (active && lane < deg) {
    sig_nbr[beg + lane] = x;
    t = sig_term(x, lane, seed);
  }
#pragma unroll
  for (int j = G >> 1; j > 0; j >>= 1) t += __shfl_xor_sync(0xffffffffu, t, j);
  if (active && lane == 0) {
    unsigned long long key = sig_final(degen ? 0ULL : t, lab_in[v], deg, seed);
    slot_of[v] = (int)ht_insert(ht_keys, ht_rep, ht_mask, key, v);
  }
}

// K1a': ONE THREAD per vertex for degree <= 8 (the common case of sparse graph sets:
// molecules, ER graphs with mean degree 4).  All neighbour ids and then all neighbour
// labels are loaded as independent requests, sorted with a fixed 19-comparator network
// held in registers, hashed, and inserted.  8x fewer warps than the 8-lane version and
// one dependent memory round trip less.
#define GK_CSWAP(a, b) { const int _lo = min(a, b); const int _hi = max(a, b); a = _lo; b = _hi; }
__global__ void __launch_bounds__(256)
wl_sig_thread8(int V, const int* __restrict__ row_ptr, const int* __restrict__ col_idx,
               const int* __restrict__ lab_in, int* __restrict__ sig_nbr, unsigned long long seed, int degen,
               unsigned long long* ht_keys, int* ht_rep, unsigned ht_mask, int* __restrict__ slot_of) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  const int beg = row_ptr[v];
  const int deg = row_ptr[v + 1] - beg;
  if (deg > 8) return;  // handled by wl_sig_large
  int nb[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) nb[i] = i < deg ? col_idx[beg + i] : -1;
  int x0, x1, x2, x3, x4, x5, x6, x7;
  x0 = nb[0] >= 0 ? lab_in[nb[0]] : 0x7fffffff;
  x1 = nb[1] >= 0 ? lab_in[nb[1]] : 0x7fffffff;
  x2 = nb[2] >= 0 ? lab_in[nb[2]] : 0x7fffffff;
  x3 = nb[3] >= 0 ? lab_in[nb[3]] : 0x7fffffff;
  x4 = nb[4] >= 0 ? lab_in[nb[4]] : 0x7fffffff;
  x5 = nb[5] >= 0 ? lab_in[nb[5]] : 0x7fffffff;
  x6 = nb[6] >= 0 ? lab_in[nb[6]] : 0x7fffffff;
  x7 = nb[7] >= 0 ? lab_in[nb[7]] : 0x7fffffff;
  const int own = lab_in[v];
  // optimal 8-input sorting network (19 compare-exchanges)
  GK_CSWAP(x0, x1) GK_CSWAP(x2, x3) GK_CSWAP(x4, x5) GK_CSWAP(x6, x7)
  GK_CSWAP(x0, x2) GK_CSWAP(x1, x3) GK_CSWAP(x4, x6) GK_CSWAP(x5, x7)
  GK_CSWAP(x1, x2) GK_CSWAP(x5, x6) GK_CSWAP(x0, x4) GK_CSWAP(x3, x7)
  GK_CSWAP(x1, x5) GK_CSWAP(x2, x6)
  GK_CSWAP(x1, x4) GK_CSWAP(x3, x6)
  GK_CSWAP(x2, x4) GK_CSWAP(x3, x5)
  GK_CSWAP(x3, x4)
  const int xs[8] = {x0, x1, x2, x3, x4, x5, x6, x7};
  unsigned long long t = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    if (i < deg) {
      sig_nbr[beg + i] = xs[i];
      t += sig_term(xs[i], i, seed);
    }
  }
  const unsigned long long key = sig_final(degen ? 0ULL : t, own, deg, seed);
  slot_of[v] = (int)ht_insert(ht_keys, ht_rep, ht_mask, key, v);
}

// K1b: one warp per high-degree vertex; the neighbour labels are sorted in place in
// the vertex's own segment of sig_nbr with an all-ascending bitonic network (valid
// for any length: compare-exchanges with the virtual +inf tail are no-ops).
__global__ void __launch_bounds__(256)
wl_sig_large(int n_large, const int* __restrict__ large_list, const int* __restrict__ row_ptr,
             const int* __restrict__ col_idx, const int* __restrict__ lab_in, int* sig_nbr,
             unsigned long long seed, int degen, unsigned long long* ht_keys, int* ht_rep, unsigned ht_mask,
             int* __restrict__ slot_of) {
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= n_large) return;
  const int v = large_list[w];
  const int beg = row_ptr[v];
  const int deg = row_ptr[v + 1] - beg;
  int* seg = sig_nbr + beg;
  unsigned long long t = 0;
  if (deg <= 32) {  // one element per lane: bitonic sort in registers
    int x = lane < deg ? lab_in[col_idx[beg + lane]] : 0x7fffffff;
#pragma unroll
    for (int k = 2; k <= 32; k <<= 1) {
#pragma unroll
      for (int j = k >> 1; j > 0; j >>= 1) {
        int y = __shfl_xor_sync(0xffffffffu, x, j);
        bool up = (lane & k) == 0;
        bool lower = (lane & j) == 0;
        x = (lower == up) ? min(x, y) : max(x, y);
      }
    }
    if (lane < deg) {
      seg[lane] = x;
      t = sig_term(x, lane, seed);
    }
  } else {
    for (int i = lane; i < deg; i += 32) seg[i] = lab_in[col_idx[beg + i]];
    __syncwarp();
    int n2 = 1;
    while (n2 < deg) n2 <<= 1;
    for (int k = 2; k <= n2; k <<= 1) {
      for (int i = lane; i < deg; i += 32) {
        int p = i ^ (k - 1);
        if (p > i && p < deg) {
          int a = seg[i], b = seg[p];
          if (a > b) { seg[i] = b; seg[p] = a; }
        }
      }
      __syncwarp();
      for (int j = k >> 2; j > 0; j >>= 1) {
        for (int i = lane; i < deg; i += 32) {
          int p = i ^ j;
          if (p > i && p < deg) {
            int a = seg[i], b = seg[p];
            if (a > b) { seg[i] = b; seg[p] = a; }
          }
        }
        __syncwarp();
      }
    }
    for (int i = lane; i < deg; i += 32) t += sig_term(seg[i], i, seed);
  }
#pragma unroll
  for (int j = 16; j > 0; j >>= 1) t += __shfl_xor_sync(0xffffffffu, t, j);
  if (lane == 0) {
    unsigned long long key = sig_final(degen ? 0ULL : t, lab_in[v], deg, seed);
    slot_of[v] = (int)ht_insert(ht_keys, ht_rep, ht_mask, key, v);
  }
}

// ---------------------------------------------------------------------------
// block-wide exclusive scan helper (blockDim.x == 256)
__device__ __forceinline__ int block_exclusive_scan_256(int x, int* total) {
  __shared__ int warp_sums[8];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int incl = x;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    int y = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl += y;
  }
  if (lane == 31) warp_sums[wid] = incl;
  __syncthreads();
  if (wid == 0) {
    int s = lane < 8 ? warp_sums[lane] : 0;
#pragma unroll
    for (int d = 1; d < 8; d <<= 1) {
      int y = __shfl_up_sync(0xffffffffu, s, d);
      if (lane >= d) s += y;
    }
    if (lane < 8) warp_sums[lane] = s;
  }
  __syncthreads();
  int off = wid ? warp_sums[wid - 1] : 0;
  *total = warp_sums[7];
  __syncthreads();
  return off + incl - x;
}

// K2a: resolve each vertex to the representative (smallest vertex id) of its hash
// slot and verify the full signature against it.  flags[v] = 1 iff v is a
// representative, i.e. the first occurrence of a new compressed label.
__global__ void __launch_bounds__(256)
wl_resolve(int V, const int* __restrict__ row_ptr, const int* __restrict__ lab_in,
           const int* __restrict__ sig_nbr, const int* __restrict__ ht_rep, int* slot_of,
           int* __restrict__ flags, int* __restrict__ block_sums, DevScalars* sc) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  int f = 0;
  if (v < V) {
    const int r = ht_rep[slot_of[v]];
    slot_of[v] = r;
    f = (r == v);
    if (!f) {
      const int bv = row_ptr[v], dv = row_ptr[v + 1] - bv;
      const int br = row_ptr[r], dr = row_ptr[r + 1] - br;
      bool same = (dv == dr) && (lab_in[v] == lab_in[r]);
      for (int i = 0; same && i < dv; ++i) same = sig_nbr[bv + i] == sig_nbr[br + i];
      if (!same) atomicOr(&sc->collision, 1u);
    }
    flags[v] = f;
  }
  int total;
  block_exclusive_scan_256(f, &total);
  if (threadIdx.x == 0) block_sums[blockIdx.x] = total;
}

// exclusive scan of block_sums in place by ONE block; writes the grand total to
// *dim_out and chains the running column base (*base_out = *base_in + total).
__global__ void __launch_bounds__(256)
scan_block_sums(int nb, int* block_sums, long long* dim_out, const long long* base_in,
                long long* base_out) {
  __shared__ int carry_s;
  if (threadIdx.x == 0) carry_s = 0;
  __syncthreads();
  for (int start = 0; start < nb; start += 256) {
    const int i = start + threadIdx.x;
    int x = i < nb ? block_sums[i] : 0;
    int total;
    int ex = block_exclusive_scan_256(x, &total);
    const int carry = carry_s;
    if (i < nb) block_sums[i] = carry + ex;
    __syncthreads();
    if (threadIdx.x == 0) carry_s = carry + total;
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    if (dim_out) *dim_out = carry_s;
    if (base_out) *base_out = (base_in ? *base_in : 0) + carry_s;
  }
}

// sum of block_sums[0 .. blockIdx.x) computed by the block itself (replaces a separate
// single-block scan launch; the array has V/256 entries and lives in L2)
__device__ __forceinline__ long long block_prefix_of_sums(const int* __restrict__ block_sums) {
  __shared__ long long red[8];
  long long s = 0;
  for (int i = threadIdx.x; i < (int)blockIdx.x; i += blockDim.x) s += block_sums[i];
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) s += __shfl_xor_sync(0xffffffffu, s, d);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  long long tot = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) tot += red[i];
  __syncthreads();
  return tot;
}

// K2b: representatives receive their dense id (rank among representatives).  The last
// block also publishes the level's label count and the next level's first column.
__global__ void __launch_bounds__(256)
wl_assign(int V, int level, const int* __restrict__ flags, const int* __restrict__ block_sums,
          int* __restrict__ lab_out, DevScalars* sc) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  const int f = v < V ? flags[v] : 0;
  int total;
  const int ex = block_exclusive_scan_256(f, &total);
  const long long base = block_prefix_of_sums(block_sums);
  if (f) lab_out[v] = (int)base + ex;
  if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) {
    sc->level_dims[level] = base + total;
    sc->level_base[level + 1] = sc->level_base[level] + base + total;
  }
}

// Per-column / per-graph statistics maintained while the feature block is being filled,
// so that no extra pass over the (4x over-provisioned) table is needed afterwards.
struct FeatStats {
  unsigned* colcnt;            // graphs holding the column (saturating at COL_CAP)
  unsigned long long* diag;    // per graph: sum of squared counts (exact self similarity)
  unsigned* part_max;          // per-CTA partials (no same-address atomics in the hot path):
  unsigned* part_new;          //   largest count seen / entries created by the CTA
  DevScalars* sc;
};
constexpr unsigned COL_CAP = 1u << 13;  // column counters saturate here ("certainly head")

// (graph, column) -> count.  `base` selects a sub-table (one per WL level) so that the
// table being hammered by a level's insert pass stays L2-resident.  Returns the count
// before this insertion; *is_new is set when the (graph, column) entry was created.
__device__ __forceinline__ unsigned ft_add(unsigned long long* keys, unsigned* cnt, unsigned mask,
                                           unsigned long long key, unsigned inc, const FeatStats& st,
                                           bool* is_new, size_t base = 0) {
  unsigned slot = (unsigned)(mix64(key) >> 17) & mask;
  for (int probe = 0; probe < 8192; ++probe) {
    unsigned long long prev = __ldcg(&keys[base + slot]);
    bool created = false;
    if (prev == EMPTY64) {
      prev = atomicCAS(&keys[base + slot], EMPTY64, key);
      created = prev == EMPTY64;
    }
    if (created || prev == key) {
      const unsigned old = atomicAdd(&cnt[base + slot], inc);
      if (created) {
        const unsigned c = (unsigned)key;
        if (__ldcg(&st.colcnt[c]) < COL_CAP) atomicAdd(&st.colcnt[c], 1u);
      }
      *is_new = created;
      return old;
    }
    slot = (slot + 1) & mask;
  }
  atomicOr(&st.sc->ft_overflow, 1u);  // table too small: the host grows it and repeats the pass
  *is_new = false;
  return 0;
}

// Block-wide bookkeeping after every thread has done (at most) one ft_add with inc == 1:
//   diag[g] += (old+1)^2 - old^2 = 2*old + 1, aggregated over runs of equal g inside a warp
//   (vertices of a graph are contiguous); max count and entry count go to per-CTA partials.
__device__ __forceinline__ void ft_account(bool did, int g, unsigned old, bool is_new, const FeatStats& st,
                                           size_t part_index) {
  const int lane = threadIdx.x & 31;
  unsigned long long val = did ? 2ULL * old + 1ULL : 0ULL;
  const int gg = did ? g : -1;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const unsigned long long y = __shfl_down_sync(0xffffffffu, val, d);
    const int gy = __shfl_down_sync(0xffffffffu, gg, d);
    if (lane + d < 32 && gy == gg) val += y;
  }
  const int gprev = __shfl_up_sync(0xffffffffu, gg, 1);
  if (did && (lane == 0 || gprev != gg)) atomicAdd(&st.diag[g], val);
  __shared__ unsigned s_mx[8], s_n[8];
  unsigned mx = did ? old + 1 : 0, n = is_new ? 1u : 0u;
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, d));
    n += __shfl_xor_sync(0xffffffffu, n, d);
  }
  if (lane == 0) { s_mx[threadIdx.x >> 5] = mx; s_n[threadIdx.x >> 5] = n; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < 8; ++w) { mx = max(mx, s_mx[w]); n += s_n[w]; }
    st.part_max[part_index] = mx;
    st.part_new[part_index] = n;
  }
}

// K2c + K3a: every vertex takes the id of its representative; the (graph, column)
// pair is counted into the sparse feature block (vertex_histogram.py:107-122).
__global__ void __launch_bounds__(256)
wl_gather_insert(int V, int level, const int* __restrict__ rep_of, int* lab_out,
                 const int* __restrict__ vgraph, FeatStats st,
                 unsigned long long* ft_keys, unsigned* ft_cnt, unsigned ft_mask) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  bool did = false, is_new = false;
  int g = 0;
  unsigned old = 0;
  if (v < V) {
    const int r = rep_of[v];
    const int id = lab_out[r];
    if (r != v) lab_out[v] = id;
    const unsigned long long col = (unsigned long long)(st.sc->level_base[level] + id);
    g = vgraph[v];
    old = ft_add(ft_keys, ft_cnt, ft_mask, ((unsigned long long)(unsigned)g << 32) | col, 1u, st, &is_new,
                 (size_t)level * ((size_t)ft_mask + 1));
    did = true;
  }
  ft_account(did, g, old, is_new, st, (size_t)level * gridDim.x + blockIdx.x);
}

__global__ void __launch_bounds__(256)
wl_insert_level0(int V, const int* __restrict__ lab, const int* __restrict__ vgraph,
                 unsigned long long* ft_keys, unsigned* ft_cnt, unsigned ft_mask, FeatStats st) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  bool did = false, is_new = false;
  int g = 0;
  unsigned old = 0;
  if (v < V) {
    g = vgraph[v];
    old = ft_add(ft_keys, ft_cnt, ft_mask,
                 ((unsigned long long)(unsigned)g << 32) | (unsigned long long)(unsigned)lab[v], 1u, st, &is_new);
    did = true;
  }
  ft_account(did, g, old, is_new, st, blockIdx.x);
}

// CSR statistics + validation on the device (replaces host loops over V and E in gk_pack_csr):
// out[0..4] degree histogram (<=4, <=8, <=16, <=32, more), out[5] max degree, out[6] error bits
// (1 = negative degree, 2 = neighbour outside its graph, 4 = negative label), out[7] max label.
__global__ void __launch_bounds__(256)
pack_scan(int V, int E, const int* __restrict__ graph_ptr, const int* __restrict__ vgraph,
          const int* __restrict__ row_ptr, const int* __restrict__ col_idx, const int* __restrict__ labels,
          int* out) {
  __shared__ int sh[8];
  if (threadIdx.x < 8) sh[threadIdx.x] = 0;
  __syncthreads();
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v < V) {
    const int b = row_ptr[v], d = row_ptr[v + 1] - b;
    int err = (d < 0 || b < 0 || (long long)b + d > E) ? 1 : 0;
    const int g = vgraph[v];
    const int v0 = graph_ptr[g], v1 = graph_ptr[g + 1];
    for (int e = 0; e < d && !err; ++e) {
      const int w = col_idx[b + e];
      if (w < v0 || w >= v1) err |= 2;
    }
    int lab = 0;
    if (labels) { lab = labels[v]; if (lab < 0) err |= 4; }
    atomicAdd(&sh[(d > 4) + (d > 8) + (d > 16) + (d > 32)], 1);
    atomicMax(&sh[5], d);
    if (err) atomicOr(&sh[6], err);
    atomicMax(&sh[7], lab);
  }
  __syncthreads();
  if (threadIdx.x < 5 && sh[threadIdx.x]) atomicAdd(&out[threadIdx.x], sh[threadIdx.x]);
  if (threadIdx.x == 5) atomicMax(&out[5], sh[5]);
  if (threadIdx.x == 6 && sh[6]) atomicOr(&out[6], sh[6]);
  if (threadIdx.x == 7) atomicMax(&out[7], sh[7]);
}

// edge weights: out[8] bit 1 = some weight != 1, bit 2 = negative or NaN weight
__global__ void __launch_bounds__(256)
pack_scan_weights(long long E, const double* __restrict__ w, int* out) {
  int f = 0;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < E; e += (long long)gridDim.x * blockDim.x) {
    const double x = w[e];
    if (!(x >= 0.0)) f |= 2;
    if (x != 1.0) f |= 1;
  }
  f = __reduce_or_sync(0xffffffffu, f);
  if ((threadIdx.x & 31) == 0 && f) atomicOr(&out[8], f);
}

// vertices whose degree exceeds the chosen lane width -> list for wl_sig_large (order irrelevant)
__global__ void __launch_bounds__(256)
pack_large_list(int V, const int* __restrict__ row_ptr, int width, int* __restrict__ list, int* counter) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  if (row_ptr[v + 1] - row_ptr[v] > width) list[atomicAdd(counter, 1)] = v;
}

// vertex -> graph id by binary search in graph_ptr
__global__ void __launch_bounds__(256)
fill_vgraph(int V, int N, const int* __restrict__ graph_ptr, int* __restrict__ vgraph) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  int lo = 0, hi = N;  // find g with graph_ptr[g] <= v < graph_ptr[g+1]
  while (hi - lo > 1) {
    int mid = (lo + hi) >> 1;
    if (graph_ptr[mid] <= v) lo = mid; else hi = mid;
  }
  vgraph[v] = lo;
}

}  // namespace gk
