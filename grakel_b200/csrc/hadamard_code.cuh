// HadamardCode relabelling (hadamard_code.py:186-215) on the device, sm_90a.
//
// Every vertex carries a vector of W = 2^ceil(log2 nl) int64 entries, stored as u64 so that the additions wrap like
// numpy's int64 arithmetic without undefined behaviour.  Level 0 is row `label` of Sylvester's Hadamard matrix,
// H[r, c] = (-1)^popcount(r & c), computed in place (H is never materialised); level i >= 1 adds the level-(i-1)
// vectors of a vertex's out-neighbours to its own, a self-loop counting once more.  Skipped vertices (labelled, but not
// keys of the edge dictionary) have no vector at levels >= 1.
//
// Classes are exact vector equality: a vector's 64-bit hash h = sum_c s_c z_c (mod 2^64, seeded odd z_c) goes into an
// open-addressing table whose slots keep their smallest vertex as representative, and every vertex then compares its
// full vector with its representative's (hc_verify).  A mismatch sets DevScalars::collision and the host repeats the
// pass with another seed.  The dense class ids and the (graph, column) counts reuse the WL multi-kernel path's
// wl_assign and ft_add (wl.cuh), so the result is an ordinary FK_WL feature block.
//
// Thread shape: a group of T = min(W, 32) lanes per vertex, lane c handling entries c, c + T, ...; a warp holds 32 / T
// vertices, so the common W = 8 reads 64 contiguous bytes per vertex and neighbour with 8 lanes.
#pragma once
#include "common.cuh"
#include "wl.cuh"

namespace gk {

constexpr int HC_THREADS = 256;

struct HcShape {
  int V;
  int lgW, lgT;  // W = 2^lgW entries per vector, T = 2^lgT lanes per vertex
};

__device__ __forceinline__ unsigned long long hc_group_sum(unsigned long long x, int T) {
  for (int d = T >> 1; d > 0; d >>= 1) x += __shfl_xor_sync(0xffffffffu, x, d, T);
  return x;
}

// slot of hash `hv` in the level's table: key install + smallest vertex as representative
__device__ __forceinline__ void hc_insert(unsigned long long hv, int v, unsigned long long* ht_keys, int* ht_rep,
                                          unsigned mask, int* slot_of, DevScalars* sc) {
  const unsigned long long key = hv == EMPTY64 ? EMPTY64 - 1 : hv;  // the empty marker is not a key
  unsigned slot = (unsigned)(mix64(key) >> 20) & mask;
  for (unsigned probe = 0; probe <= mask; ++probe) {
    unsigned long long prev = __ldcg(&ht_keys[slot]);
    if (prev == EMPTY64) prev = atomicCAS(&ht_keys[slot], EMPTY64, key);
    if (prev == EMPTY64 || prev == key) {
      atomicMin(&ht_rep[slot], v);
      slot_of[v] = (int)slot;
      return;
    }
    slot = (slot + 1) & mask;
  }
  atomicOr(&sc->ft_overflow, 4u);  // cannot happen at load <= 0.5
}

// Level 0: S[v] = H[label(v)], hashed and inserted (ht_keys null: vectors only, for gk_hc_vectors)
__global__ void __launch_bounds__(HC_THREADS)
hc_level0(HcShape s, const int* __restrict__ labels, const unsigned long long* __restrict__ z, unsigned long long* S,
          unsigned long long* ht_keys, int* ht_rep, unsigned mask, int* slot_of, DevScalars* sc) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int T = 1 << s.lgT, W = 1 << s.lgW;
  const int v = (int)(t >> s.lgT), lane = (int)(t & (T - 1));
  const bool live = v < s.V;
  unsigned long long hv = 0;
  if (live) {
    const unsigned r = (unsigned)labels[v];
    unsigned long long* row = S + ((size_t)v << s.lgW);
    for (int c = lane; c < W; c += T) {
      const unsigned long long x = (__popc(r & (unsigned)c) & 1) ? ~0ULL : 1ULL;
      row[c] = x;
      hv += x * __ldg(&z[c]);
    }
  }
  hv = hc_group_sum(hv, T);
  if (live && lane == 0 && ht_keys) hc_insert(hv, v, ht_keys, ht_rep, mask, slot_of, sc);
}

// Level i >= 1: S_out[v] = S_in[v] + sum over out-neighbours q of S_in[q]; skipped vertices get a zero vector
__global__ void __launch_bounds__(HC_THREADS)
hc_step(HcShape s, const int* __restrict__ row_ptr, const int* __restrict__ col_idx,
        const unsigned char* __restrict__ skip, const unsigned long long* __restrict__ z,
        const unsigned long long* __restrict__ S_in, unsigned long long* __restrict__ S_out,
        unsigned long long* ht_keys, int* ht_rep, unsigned mask, int* slot_of, DevScalars* sc) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int T = 1 << s.lgT, W = 1 << s.lgW;
  const int v = (int)(t >> s.lgT), lane = (int)(t & (T - 1));
  const bool live = v < s.V && !(skip && skip[v]);
  unsigned long long hv = 0;
  if (v < s.V) {
    unsigned long long* out = S_out + ((size_t)v << s.lgW);
    if (live) {
      const int b = row_ptr[v], e = row_ptr[v + 1];
      for (int c = lane; c < W; c += T) {
        unsigned long long x = S_in[((size_t)v << s.lgW) + c];
        for (int k = b; k < e; ++k) x += S_in[((size_t)__ldg(&col_idx[k]) << s.lgW) + c];
        out[c] = x;
        hv += x * __ldg(&z[c]);
      }
    } else {
      for (int c = lane; c < W; c += T) out[c] = 0ULL;
    }
  }
  hv = hc_group_sum(hv, T);
  if (live && lane == 0 && ht_keys) hc_insert(hv, v, ht_keys, ht_rep, mask, slot_of, sc);
}

// Every live vertex takes its slot's representative (slot_of[v] <- rep) and compares its full vector with it;
// flags[v] = 1 iff v is a representative.  A mismatch is a hash collision.
__global__ void __launch_bounds__(HC_THREADS)
hc_verify(HcShape s, const unsigned char* __restrict__ skip, const unsigned long long* __restrict__ S,
          const int* __restrict__ ht_rep, int* slot_of, int* __restrict__ flags, DevScalars* sc) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int T = 1 << s.lgT, W = 1 << s.lgW;
  const int v = (int)(t >> s.lgT), lane = (int)(t & (T - 1));
  const bool live = v < s.V && !(skip && skip[v]);
  int r = v;
  if (live) r = ht_rep[slot_of[v]];
  bool differ = false;
  if (live && r != v)
    for (int c = lane; c < W; c += T) differ |= S[((size_t)v << s.lgW) + c] != S[((size_t)r << s.lgW) + c];
  if (differ) atomicOr(&sc->collision, 1u);
  if (v < s.V && lane == 0) {
    if (live) slot_of[v] = r;
    flags[v] = live && r == v;
  }
}

// representatives per block of 256 vertices (the block_sums wl_assign reads)
__global__ void __launch_bounds__(256)
hc_flag_sums(int V, const int* __restrict__ flags, int* __restrict__ block_sums) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  int total;
  block_exclusive_scan_256(v < V ? flags[v] : 0, &total);
  if (threadIdx.x == 0) block_sums[blockIdx.x] = total;
}

// ft_account for a block in which some vertices count nothing: a skipped vertex keeps its graph id in the warp's
// run of equal graphs (with a zero increment), so that the run-wise sum of the self-similarity increments only ever
// adds contiguous lanes -- a -1 in the middle of a graph's run would let lanes on both sides count one stretch twice
__device__ __forceinline__ void hc_account(bool in_range, bool did, int g, unsigned old, bool is_new, const FeatStats& st,
                                           size_t part_index) {
  const int lane = threadIdx.x & 31;
  unsigned long long val = did ? 2ULL * old + 1ULL : 0ULL;
  const int gg = in_range ? g : -1;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const unsigned long long y = __shfl_down_sync(0xffffffffu, val, d);
    const int gy = __shfl_down_sync(0xffffffffu, gg, d);
    if (lane + d < 32 && gy == gg) val += y;
  }
  const int gprev = __shfl_up_sync(0xffffffffu, gg, 1);
  if (in_range && val && (lane == 0 || gprev != gg)) atomicAdd(&st.diag[g], val);
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

// every live vertex takes its representative's dense id (-1 for a skipped vertex) and, unless ft_keys is null (the
// ShortestPath base only needs the ids), counts (graph, level_base + id) into the level's sub-table of the feature
// block, as wl_gather_insert does
__global__ void __launch_bounds__(256)
hc_gather_insert(int V, int level, const unsigned char* __restrict__ skip, const int* __restrict__ rep_of,
                 int* lab_out, const int* __restrict__ vgraph, FeatStats st, unsigned long long* ft_keys,
                 unsigned* ft_cnt, unsigned ft_mask) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  bool did = false, is_new = false;
  const int g = v < V ? vgraph[v] : 0;
  unsigned old = 0;
  if (v < V) {
    if (skip && skip[v]) {
      lab_out[v] = -1;
    } else {
      const int r = rep_of[v];
      const int id = lab_out[r];
      if (r != v) lab_out[v] = id;
      if (ft_keys) {
        const unsigned long long col = (unsigned long long)(st.sc->level_base[level] + id);
        old = ft_add(ft_keys, ft_cnt, ft_mask, ((unsigned long long)(unsigned)g << 32) | col, 1u, st, &is_new,
                     (size_t)level * ((size_t)ft_mask + 1));
        did = true;
      }
    }
  }
  hc_account(v < V, did, g, old, is_new, st, (size_t)level * gridDim.x + blockIdx.x);
}

}  // namespace gk
