// All WL levels in ONE persistent cooperative kernel (weisfeiler_lehman.py:199-258 +
// vertex_histogram.py:107-122 for every level), staged through shared memory.
//
// Why: the multi-kernel pipeline of wl.cuh spends each level in five latency-bound launches, far above
// its HBM floor.  Micro-benchmarks (tools/mb/wl_mb.cu) show the limit is the number of SCATTERED L2
// operations per vertex, so this kernel is organised to minimise them:
//
//   * The graphs are cut into TILES of whole graphs (<= WLF_TILE_V vertices, <= WLF_TILE_E edges);
//     each CTA owns a contiguous run of tiles.  A tile's CSR slice and labels are staged into
//     shared memory with coalesced loads; neighbour gathers, sorting and the per-graph label
//     histogram never leave shared memory.
//   * Signature dedup uses ONE packed 64-bit word per slot, {32-bit tag | representative vertex}:
//     insert = 1 L2 read + (1 CAS when the slot is empty | 1 atomicMin when the tag matches and the
//     current representative is larger | nothing).  The full signature is still verified against
//     the representative's, so the partition is exact; a tag clash only triggers the host's retry.
//   * (graph, column) counts are produced by comparing labels inside the graph in shared memory
//     (a graph never straddles a tile) and appended to a compact COO list -- no global feature
//     hash table, no per-level table clearing, and the Gram stage streams 12 B per entry instead
//     of 12 B per (4x over-provisioned) slot.
//
// A level is   [A] signatures + insert | grid barrier | [B] representative + verification + ranks
//              | grid barrier | [C] dense first-occurrence ids, labels, feature entries
// and [A] of the next level follows [C] after a __syncthreads only, because everything a tile
// needs from the previous level (labels of its own vertices) was written by the same CTA.
#pragma once
#include "common.cuh"
#include "wl.cuh"

namespace gk {

constexpr int WLF_THREADS = 1024;
constexpr int WLF_TILE_V = 4096;    // vertices per tile (u16 local indices)
constexpr int WLF_TILE_E = 16384;   // edges per tile
constexpr int WLF_VPT = WLF_TILE_V / WLF_THREADS;  // vertices per thread and tile (register batches)
constexpr int WLF_AGG = 8192;       // per-tile column -> graph-count aggregation table (shared memory)
constexpr int WLF_RANK_BITS = 20;   // rank_pack = cta << 20 | rank of the representative inside its CTA
constexpr int WLF_SMEM = (WLF_TILE_V + 1) * 4 /*rp_s*/ + 4 /*pad*/ + WLF_TILE_V * 8 /*key_s*/ + WLF_TILE_V * 4 /*lab_s*/ +
                         WLF_TILE_E * 4 /*sig_s | agg*/ + WLF_TILE_E * 2 /*col_s*/ + 16;
static_assert(WLF_AGG * 8 <= WLF_TILE_E * 4, "aggregation table must fit in the sig_s region");

struct WlFusedParams {
  int V, L;
  const int* graph_ptr;
  const int* row_ptr;
  const int* col_idx;
  const int* vgraph;
  const int* labels0;
  const int* tile_vbeg;  // [n_tiles + 1] first vertex of each tile (whole graphs)
  const int* cta_tile;   // [grid + 1] first tile of each CTA
  int* labels_all;       // [L * V]
  int* sig_nbr;          // [E] sorted neighbour labels of the current level
  int* slot_of;          // [V] hash slot, then representative vertex
  int* rank_pack;        // [V] valid for representatives
  unsigned char* single; // [V] zeroed by the host: the vertex's label of the previous level is held by no other vertex
  int* cta_count;        // [grid]
  unsigned long long* table;  // 2 x (ht_mask + 1) packed {tag, representative} words
  unsigned ht_mask;
  unsigned long long* coo_keys;  // feature entries: graph << 32 | column
  unsigned* coo_cnt;
  unsigned* barrier;  // zeroed by the host before the launch
  unsigned long long seed;
  int degen_from;     // levels >= degen_from hash (own label, degree) only (gk_selftest_wl_collision); INT_MAX = off
  FeatStats st;
  DevScalars* sc;
  long long* prof;  // optional [grid][L][16] globaltimer stamps (GRAKEL_B200_PROF), else NULL
};

__device__ __forceinline__ long long wlf_now() {
  long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
#define WLF_STAMP(level, k) \
  do { if (p.prof && tid == 0) p.prof[((size_t)b * p.L + (level)) * 16 + (k)] = wlf_now(); } while (0)

__device__ __forceinline__ void wlf_grid_sync(unsigned* bar, unsigned target) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(bar, 1u);
    unsigned seen;
    do {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(seen) : "l"(bar) : "memory");
    } while (seen < target);
    __threadfence();
  }
  __syncthreads();
}

// block-wide exclusive scan for 1024 threads; returns the exclusive prefix, *total = block sum
__device__ __forceinline__ int wlf_block_scan(int x, int* total, int* s_warp /*[32]*/) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int incl = x;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl += y;
  }
  if (lane == 31) s_warp[wid] = incl;
  __syncthreads();
  if (wid == 0) {
    int s = s_warp[lane];
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, s, d);
      if (lane >= d) s += y;
    }
    s_warp[lane] = s;
  }
  __syncthreads();
  const int off = wid ? s_warp[wid - 1] : 0;
  *total = s_warp[31];
  __syncthreads();
  return off + incl - x;
}

// ---- signature hashes (32-bit arithmetic; two independent lanes -> {tag, home slot}).
// Equal signatures have equal degree, hence always take the same code path, so the
// thread-per-vertex path (sequential over the sorted labels) and the warp path (sum of
// positional terms) may use different functions.  Exactness never depends on the hash:
// every vertex is verified against its representative and a clash makes the host retry.
__device__ __forceinline__ unsigned wlf_fmix(unsigned h) {
  h ^= h >> 16; h *= 0x85EBCA6Bu; h ^= h >> 13; h *= 0xC2B2AE35u; h ^= h >> 16;
  return h;
}
__device__ __forceinline__ unsigned long long wlf_finish(unsigned a, unsigned c, int own, int deg, unsigned long long seed) {
  a = wlf_fmix(a ^ ((unsigned)own * 0x9E3779B1u) ^ (unsigned)seed);
  c = wlf_fmix(c + (unsigned)own * 0x7FEB352Du + (unsigned)deg * 0x846CA68Bu + (unsigned)(seed >> 32));
  return (((unsigned long long)a << 32) | c) >> 1;  // never EMPTY64
}
__device__ __forceinline__ void wlf_seq_step(unsigned& a, unsigned& c, int x) {
  a = (a ^ (unsigned)x) * 0x9E3779B1u; a ^= a >> 15;
  c = (c + (unsigned)x) * 0x85EBCA77u; c ^= c >> 13;
}
__device__ __forceinline__ void wlf_pos_term(unsigned& a, unsigned& c, int x, int pos, unsigned long long seed) {
  a += wlf_fmix((unsigned)x * 0x9E3779B1u + (unsigned)pos * 0x85EBCA77u + (unsigned)seed);
  c += wlf_fmix(((unsigned)x ^ 0x5bd1e995u) * 0xC2B2AE3Du + (unsigned)pos * 0x27D4EB2Fu + (unsigned)(seed >> 32));
}

// stage one tile: CSR slice (row offsets relative to the tile, neighbours as tile-local u16)
__device__ __forceinline__ void wlf_stage(const WlFusedParams& p, int v0, int nv, int e0, int ne, const int* lab_src,
                                          int* rp_s, unsigned short* col_s, int* lab_s, bool with_csr) {
  const int tid = threadIdx.x;
  if (with_csr) {
    for (int i = tid; i <= nv; i += WLF_THREADS) rp_s[i] = p.row_ptr[v0 + i] - e0;
    for (int k = tid; k < ne; k += WLF_THREADS) col_s[k] = (unsigned short)(p.col_idx[e0 + k] - v0);
  }
  if (lab_src)
    for (int i = tid; i < nv; i += WLF_THREADS) lab_s[i] = lab_src[v0 + i];
}

// Feature entries of one tile from the labels in lab_s: vertex i emits (graph, base + label, count)
// iff it is the first vertex of its graph carrying that label (labels compared inside the graph in
// shared memory).  One COO reservation per tile; the per-column graph counts are aggregated in a
// shared-memory table first, so a column shared by every graph costs one global atomic per tile.
__device__ __forceinline__ void wlf_emit(const WlFusedParams& p, int v0, int nv, const int* lab_s, unsigned* agg,
                                         long long base, size_t coo_off, int* s_warp, unsigned& mx, unsigned& n_new,
                                         const unsigned char* single = nullptr) {
  const int tid = threadIdx.x, lane = tid & 31;
  for (int s = tid; s < WLF_AGG * 2; s += WLF_THREADS) agg[s] = (s & 1) ? 0u : 0xFFFFFFFFu;  // {column, graphs}
  int g[WLF_VPT], l[WLF_VPT], gs[WLF_VPT], ge[WLF_VPT];
  unsigned cnt[WLF_VPT];
  bool emit[WLF_VPT];
#pragma unroll
  for (int k = 0; k < WLF_VPT; ++k) {
    const int i = tid + k * WLF_THREADS;
    g[k] = i < nv ? p.vgraph[v0 + i] : -1;
  }
#pragma unroll
  for (int k = 0; k < WLF_VPT; ++k) {
    gs[k] = ge[k] = 0;
    if (g[k] >= 0) { gs[k] = p.graph_ptr[g[k]] - v0; ge[k] = p.graph_ptr[g[k] + 1] - v0; }
  }
  int n_emit = 0;
#pragma unroll
  for (int k = 0; k < WLF_VPT; ++k) {
    const int i = tid + k * WLF_THREADS;
    cnt[k] = 0;
    emit[k] = false;
    l[k] = 0;
    if (g[k] >= 0 && single && single[v0 + i]) {  // label unique in the whole data set: one entry, count 1
      l[k] = lab_s[i];
      cnt[k] = 1;
      emit[k] = true;
      n_emit += 1;
    } else if (g[k] >= 0) {
      l[k] = lab_s[i];
      bool first = true;
      for (int u = gs[k]; u < ge[k]; ++u) {
        const bool same = lab_s[u] == l[k];
        cnt[k] += same ? 1u : 0u;
        first = first && !(same && u < i);
      }
      emit[k] = first;
      n_emit += first ? 1 : 0;
    }
  }
  // Every (tile, level) owns a fixed region of the COO arrays, [coo_off, coo_off + nv): at most one
  // entry per vertex, so no global reservation (an atomic round trip that stalls the whole CTA) is
  // needed; the unused remainder is filled with EMPTY64 keys, which every consumer skips.
  int total;
  int ex = wlf_block_scan(n_emit, &total, s_warp);  // also orders the agg initialisation before its use
  const size_t off = coo_off;
  for (int i = total + tid; i < nv; i += WLF_THREADS) p.coo_keys[off + i] = EMPTY64;
#pragma unroll
  for (int k = 0; k < WLF_VPT; ++k) {
    if (emit[k]) {
      const unsigned col = (unsigned)(base + l[k]);
      p.coo_keys[off + ex] = ((unsigned long long)(unsigned)g[k] << 32) | col;
      p.coo_cnt[off + ex] = cnt[k];
      ++ex;
      mx = max(mx, cnt[k]);
      n_new += 1u;
      unsigned slot = (col * 0x9E3779B1u >> 12) & (WLF_AGG - 1);
      while (true) {
        unsigned prev = agg[2 * slot];
        if (prev == 0xFFFFFFFFu) prev = atomicCAS(&agg[2 * slot], 0xFFFFFFFFu, col);
        if (prev == 0xFFFFFFFFu || prev == col) { atomicAdd(&agg[2 * slot + 1], 1u); break; }
        slot = (slot + 1) & (WLF_AGG - 1);
      }
    }
    // exact self similarity: sum of squared counts per graph (runs of equal g inside the warp)
    unsigned long long val = emit[k] ? (unsigned long long)cnt[k] * cnt[k] : 0ULL;
    const int gg = g[k];
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const unsigned long long y = __shfl_down_sync(0xffffffffu, val, d);
      const int gy = __shfl_down_sync(0xffffffffu, gg, d);
      if (lane + d < 32 && gy == gg) val += y;
    }
    const int gprev = __shfl_up_sync(0xffffffffu, gg, 1);
    if (gg >= 0 && (lane == 0 || gprev != gg) && val) atomicAdd(&p.st.diag[gg], val);
  }
  __syncthreads();
  for (int s = tid; s < WLF_AGG; s += WLF_THREADS) {
    const unsigned col = agg[2 * s];
    if (col != 0xFFFFFFFFu) atomicAdd(&p.st.colcnt[col], agg[2 * s + 1]);
  }
  __syncthreads();  // agg is reused by the next tile
}

// Vertices whose previous label is a singleton class (no other vertex of the data set carries it) are not hashed,
// inserted or verified again -- their next label is necessarily a singleton too (the signature contains the own
// label) -- and their feature entry is (graph, column, 1) without the in-graph count.  From level 3 on that is 96 % of
// the vertices of BASELINE config 2.  The table word carries a "single" bit below the 30-bit tag: the installing CAS
// sets it, the first matching vertex clears it with the atomicMin that also elects the smaller representative.
__global__ void __launch_bounds__(WLF_THREADS, 1)
wl_fused_kernel(WlFusedParams p) {
  extern __shared__ __align__(16) unsigned char wlf_smem[];
  int* rp_s = reinterpret_cast<int*>(wlf_smem);
  unsigned long long* key_s = reinterpret_cast<unsigned long long*>(rp_s + (WLF_TILE_V + 2));
  int* lab_s = reinterpret_cast<int*>(key_s + WLF_TILE_V);
  int* sig_s = lab_s + WLF_TILE_V;
  unsigned* agg = reinterpret_cast<unsigned*>(sig_s);  // phase [C] only
  unsigned short* col_s = reinterpret_cast<unsigned short*>(sig_s + WLF_TILE_E);
  __shared__ int s_warp[32];
  __shared__ int s_prefix[1024];  // exclusive scan of the CTA counts (grid <= 1024)
  __shared__ unsigned s_red[64];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int G = gridDim.x, b = blockIdx.x;
  const int t_beg = p.cta_tile[b], t_end = p.cta_tile[b + 1];
  const int V = p.V;
  const size_t ht_cap = (size_t)p.ht_mask + 1;
  unsigned n_sync = 0;
  long long level_base = 0;  // first column of the current level (uniform across the grid)
  unsigned mx = 0, n_new = 0;
  WLF_STAMP(0, 0);

  // publish the per-CTA partials of a level (max count, created entries)
  auto flush_partials = [&](int level) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
      mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, d));
      n_new += __shfl_xor_sync(0xffffffffu, n_new, d);
    }
    if (lane == 0) { s_red[wid] = mx; s_red[32 + wid] = n_new; }
    __syncthreads();
    if (tid == 0) {
      unsigned m = 0, n = 0;
      for (int w = 0; w < 32; ++w) { m = max(m, s_red[w]); n += s_red[32 + w]; }
      p.st.part_max[(size_t)level * G + b] = m;
      p.st.part_new[(size_t)level * G + b] = n;
    }
    mx = 0;
    n_new = 0;
    __syncthreads();
  };

  // ---- level 0: labels as given
  for (int t = t_beg; t < t_end; ++t) {
    const int v0 = p.tile_vbeg[t], nv = p.tile_vbeg[t + 1] - v0;
    wlf_stage(p, v0, nv, 0, 0, p.labels0, rp_s, col_s, lab_s, false);
    for (int i = tid; i < nv; i += WLF_THREADS) p.labels_all[v0 + i] = p.labels0[v0 + i];
    __syncthreads();
    wlf_emit(p, v0, nv, lab_s, agg, 0, (size_t)v0, s_warp, mx, n_new);
  }
  level_base = p.sc->level_base[1];  // = number of level-0 labels (set by the host)
  flush_partials(0);
  WLF_STAMP(0, 6);

  for (int lv = 1; lv < p.L; ++lv) {
    const int* lab_in = p.labels_all + (size_t)(lv - 1) * V;
    int* lab_out = p.labels_all + (size_t)lv * V;
    unsigned long long* tab = p.table + (size_t)(lv & 1) * ht_cap;

    // ---------------- [A] signatures + insert
    WLF_STAMP(lv, 0);
    for (int t = t_beg; t < t_end; ++t) {
      const int v0 = p.tile_vbeg[t], nv = p.tile_vbeg[t + 1] - v0;
      const int e0 = p.row_ptr[v0], ne = p.row_ptr[v0 + nv] - e0;
      __syncthreads();  // previous tile's shared memory is no longer read
      wlf_stage(p, v0, nv, e0, ne, lab_in, rp_s, col_s, lab_s, true);
      __syncthreads();
      WLF_STAMP(lv, 8);
      // [A1] one thread per vertex of degree <= 8: 19-comparator network in registers
      for (int i = tid; i < nv; i += WLF_THREADS) {
        const int beg = rp_s[i];
        const int deg = rp_s[i + 1] - beg;
        if (deg > 8) continue;
        if (p.single[v0 + i]) continue;
        int x0, x1, x2, x3, x4, x5, x6, x7;
        x0 = 0 < deg ? lab_s[col_s[beg + 0]] : 0x7fffffff;
        x1 = 1 < deg ? lab_s[col_s[beg + 1]] : 0x7fffffff;
        x2 = 2 < deg ? lab_s[col_s[beg + 2]] : 0x7fffffff;
        x3 = 3 < deg ? lab_s[col_s[beg + 3]] : 0x7fffffff;
        x4 = 4 < deg ? lab_s[col_s[beg + 4]] : 0x7fffffff;
        x5 = 5 < deg ? lab_s[col_s[beg + 5]] : 0x7fffffff;
        x6 = 6 < deg ? lab_s[col_s[beg + 6]] : 0x7fffffff;
        x7 = 7 < deg ? lab_s[col_s[beg + 7]] : 0x7fffffff;
        GK_CSWAP(x0, x1) GK_CSWAP(x2, x3) GK_CSWAP(x4, x5) GK_CSWAP(x6, x7)
        GK_CSWAP(x0, x2) GK_CSWAP(x1, x3) GK_CSWAP(x4, x6) GK_CSWAP(x5, x7)
        GK_CSWAP(x1, x2) GK_CSWAP(x5, x6) GK_CSWAP(x0, x4) GK_CSWAP(x3, x7)
        GK_CSWAP(x1, x5) GK_CSWAP(x2, x6)
        GK_CSWAP(x1, x4) GK_CSWAP(x3, x6)
        GK_CSWAP(x2, x4) GK_CSWAP(x3, x5)
        GK_CSWAP(x3, x4)
        const int xs[8] = {x0, x1, x2, x3, x4, x5, x6, x7};
        unsigned ha = 0x243F6A88u, hc = 0x85A308D3u;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          if (j < deg) {
            sig_s[beg + j] = xs[j];
            wlf_seq_step(ha, hc, xs[j]);
          }
        }
        const bool dg = lv >= p.degen_from;  // tests: neighbour terms left out, only the verification separates classes
        key_s[i] = wlf_finish(dg ? 0x243F6A88u : ha, dg ? 0x85A308D3u : hc, lab_s[i], deg, p.seed);
      }
      if (p.prof) { __syncthreads(); WLF_STAMP(lv, 9); }
      // [A2] higher degrees: one warp per vertex.  <= 32: one label per lane, bitonic network on
      // shuffles; above: all-ascending bitonic network in the vertex's own shared-memory segment
      // (valid for any length: exchanges with the virtual +inf tail are no-ops).
      for (int i0 = wid * 32; i0 < nv; i0 += WLF_THREADS) {
        const int iv = i0 + lane;
        bool big = iv < nv && (rp_s[iv + 1] - rp_s[iv]) > 8;
        if (big && p.single[v0 + iv]) big = false;
        unsigned m = __ballot_sync(0xffffffffu, big);
        while (m) {
          const int i = i0 + __ffs(m) - 1;
          m &= m - 1;
          const int beg = rp_s[i], deg = rp_s[i + 1] - beg;
          int* seg = sig_s + beg;
          unsigned ha = 0, hc = 0;
          if (deg <= 32) {
            int x = lane < deg ? lab_s[col_s[beg + lane]] : 0x7fffffff;
#pragma unroll
            for (int k = 2; k <= 32; k <<= 1) {
#pragma unroll
              for (int j = k >> 1; j > 0; j >>= 1) {
                const int y = __shfl_xor_sync(0xffffffffu, x, j);
                const bool up = (lane & k) == 0;
                const bool lower = (lane & j) == 0;
                x = (lower == up) ? min(x, y) : max(x, y);
              }
            }
            if (lane < deg) {
              seg[lane] = x;
              wlf_pos_term(ha, hc, x, lane, p.seed);
            }
          } else {
            for (int j = lane; j < deg; j += 32) seg[j] = lab_s[col_s[beg + j]];
            __syncwarp();
            int n2 = 1;
            while (n2 < deg) n2 <<= 1;
            for (int k = 2; k <= n2; k <<= 1) {
              for (int j = lane; j < deg; j += 32) {
                const int q = j ^ (k - 1);
                if (q > j && q < deg) {
                  const int a = seg[j], c = seg[q];
                  if (a > c) { seg[j] = c; seg[q] = a; }
                }
              }
              __syncwarp();
              for (int s = k >> 2; s > 0; s >>= 1) {
                for (int j = lane; j < deg; j += 32) {
                  const int q = j ^ s;
                  if (q > j && q < deg) {
                    const int a = seg[j], c = seg[q];
                    if (a > c) { seg[j] = c; seg[q] = a; }
                  }
                }
                __syncwarp();
              }
            }
            for (int j = lane; j < deg; j += 32) wlf_pos_term(ha, hc, seg[j], j, p.seed);
          }
#pragma unroll
          for (int s = 16; s > 0; s >>= 1) {
            ha += __shfl_xor_sync(0xffffffffu, ha, s);
            hc += __shfl_xor_sync(0xffffffffu, hc, s);
          }
          if (lane == 0) {
            const bool dg = lv >= p.degen_from;
            key_s[i] = wlf_finish(dg ? 0u : ha, dg ? 0u : hc, lab_s[i], deg, p.seed);
          }
        }
      }
      __syncthreads();
      WLF_STAMP(lv, 10);
      // [A3] insert every vertex of the tile; the (<= 4) probes of a thread are issued together
      {
        unsigned long long key[WLF_VPT], w[WLF_VPT];
        unsigned slot[WLF_VPT];
        bool act[WLF_VPT];
#pragma unroll
        for (int k = 0; k < WLF_VPT; ++k) {
          const int i = tid + k * WLF_THREADS;
          act[k] = i < nv;
          if (act[k] && p.single[v0 + i]) act[k] = false;
          key[k] = act[k] ? key_s[i] : 0ULL;
          slot[k] = (unsigned)((key[k] & 0xFFFFFFFFULL) * 0x9E3779B1ULL >> 8) & p.ht_mask;
        }
        bool any = true;
        while (any) {
          // CAS first (no read-before-CAS): a new signature costs ONE L2 round trip; an existing one
          // gets the slot's word back from the failed CAS.  Same-address CASes of a popular signature
          // serialise in the L2 slice at about one per clock, which is cheaper than a second round trip
          // for every vertex.
#pragma unroll
          for (int k = 0; k < WLF_VPT; ++k) {
            // {30-bit tag | single = 1 | vertex}
            const unsigned long long mine = (key[k] & 0xFFFFFFFF00000000ULL) | (1ULL << 32) | (unsigned)(v0 + tid + k * WLF_THREADS);
            w[k] = act[k] ? atomicCAS(&tab[slot[k]], EMPTY64, mine) : 0ULL;
          }
          any = false;
#pragma unroll
          for (int k = 0; k < WLF_VPT; ++k) {
            if (!act[k]) continue;
            const int v = v0 + tid + k * WLF_THREADS;
            if (w[k] == EMPTY64) { act[k] = false; continue; }  // the CAS installed our word
            if ((w[k] >> 33) == (key[k] >> 33)) {
              const unsigned rep = (unsigned)w[k];
              // a second member: clear the single bit and keep the smaller representative in one atomicMin
              if (((w[k] >> 32) & 1ULL) || rep > (unsigned)v)
                atomicMin(&tab[slot[k]], (key[k] & 0xFFFFFFFE00000000ULL) | (unsigned)min(rep, (unsigned)v));
              act[k] = false;
              continue;
            }
            slot[k] = (slot[k] + 1) & p.ht_mask;
            any = true;
          }
        }
#pragma unroll
        for (int k = 0; k < WLF_VPT; ++k) {
          const int i = tid + k * WLF_THREADS;
          if (i < nv) p.slot_of[v0 + i] = (int)slot[k];
        }
      }
      // sorted neighbour labels to global memory (coalesced): other CTAs verify against them
      for (int k = tid; k < ne; k += WLF_THREADS) p.sig_nbr[e0 + k] = sig_s[k];
    }
    __syncthreads();
    WLF_STAMP(lv, 1);
    wlf_grid_sync(p.barrier, (++n_sync) * (unsigned)G);
    WLF_STAMP(lv, 2);

    // ---------------- [B] representative, verification, CTA-local rank
    int carry = 0;
    for (int t = t_beg; t < t_end; ++t) {
      const int v0 = p.tile_vbeg[t], nv = p.tile_vbeg[t + 1] - v0;
      int r[WLF_VPT];
#pragma unroll
      for (int k = 0; k < WLF_VPT; ++k) {
        const int i = tid + k * WLF_THREADS;
        r[k] = i < nv ? p.slot_of[v0 + i] : 0;
      }
      bool sgl[WLF_VPT];  // the vertex's label of THIS level is a singleton class
#pragma unroll
      for (int k = 0; k < WLF_VPT; ++k) {
        const int i = tid + k * WLF_THREADS;
        sgl[k] = false;
        if (i < nv) {
          if (p.single[v0 + i]) { r[k] = v0 + i; sgl[k] = true; }  // never inserted: its own representative
          else {
            const unsigned long long word = __ldcg(&tab[r[k]]);
            r[k] = (int)(unsigned)word;
            sgl[k] = ((word >> 32) & 1ULL) && r[k] == v0 + i;
          }
        }
      }
      // verification against the representative: its CSR row and label are fetched for all (<= 4)
      // vertices of the thread at once, then up to 8 sorted neighbour labels per side in one batch
      int bv[WLF_VPT], dv[WLF_VPT], br[WLF_VPT], dr[WLF_VPT], lo[WLF_VPT], lr[WLF_VPT];
#pragma unroll
      for (int k = 0; k < WLF_VPT; ++k) {
        const int i = tid + k * WLF_THREADS;
        bv[k] = dv[k] = br[k] = dr[k] = lo[k] = lr[k] = 0;
        if (i < nv && r[k] != v0 + i) {
          bv[k] = p.row_ptr[v0 + i]; dv[k] = p.row_ptr[v0 + i + 1] - bv[k];
          br[k] = p.row_ptr[r[k]]; dr[k] = p.row_ptr[r[k] + 1] - br[k];
          lo[k] = lab_in[v0 + i]; lr[k] = __ldcg(&lab_in[r[k]]);
        }
      }
#pragma unroll
      for (int k = 0; k < WLF_VPT; ++k) {
        const int i = tid + k * WLF_THREADS;
        if (k * WLF_THREADS >= nv) break;  // uniform
        const int v = v0 + i;
        int f = 0;
        if (i < nv) {
          p.slot_of[v] = r[k];
          p.single[v] = sgl[k] ? 1 : 0;
          f = (r[k] == v);
          if (!f) {
            bool same = (dv[k] == dr[k]) && (lo[k] == lr[k]);
            if (same && dv[k] <= 8) {
              int a[8], c[8];
#pragma unroll
              for (int j = 0; j < 8; ++j) {
                a[j] = j < dv[k] ? p.sig_nbr[bv[k] + j] : 0;
                c[j] = j < dv[k] ? __ldcg(&p.sig_nbr[br[k] + j]) : 0;
              }
#pragma unroll
              for (int j = 0; j < 8; ++j) same = same && (a[j] == c[j]);
            } else {
              for (int j = 0; same && j < dv[k]; ++j) same = p.sig_nbr[bv[k] + j] == __ldcg(&p.sig_nbr[br[k] + j]);
            }
            if (!same) atomicOr(&p.sc->collision, 1u);
          }
        }
        int total;
        const int ex = wlf_block_scan(f, &total, s_warp);
        if (f) p.rank_pack[v] = (b << WLF_RANK_BITS) | (carry + ex);
        carry += total;
      }
    }
    if (tid == 0) p.cta_count[b] = carry;
    __syncthreads();
    WLF_STAMP(lv, 3);
    if (lv + 1 < p.L) {  // clear the table the next level inserts into (last read in [B] of level lv-1)
      const uint4 ones = make_uint4(0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu);
      uint4* hk = reinterpret_cast<uint4*>(p.table + (size_t)((lv + 1) & 1) * ht_cap);
      for (size_t i = (size_t)b * WLF_THREADS + tid; i < ht_cap / 2; i += (size_t)G * WLF_THREADS) hk[i] = ones;
    }
    __syncthreads();
    WLF_STAMP(lv, 4);
    wlf_grid_sync(p.barrier, (++n_sync) * (unsigned)G);
    WLF_STAMP(lv, 5);

    // ---------------- [C] dense ids, labels, feature entries
    {
      const int c = tid < G ? __ldcg(&p.cta_count[tid]) : 0;
      int total;
      const int ex = wlf_block_scan(c, &total, s_warp);
      s_prefix[tid] = ex;
      __syncthreads();
      for (int t = t_beg; t < t_end; ++t) {
        const int v0 = p.tile_vbeg[t], nv = p.tile_vbeg[t + 1] - v0;
        int r[WLF_VPT];
#pragma unroll
        for (int k = 0; k < WLF_VPT; ++k) {
          const int i = tid + k * WLF_THREADS;
          r[k] = i < nv ? p.slot_of[v0 + i] : 0;
        }
#pragma unroll
        for (int k = 0; k < WLF_VPT; ++k) {
          const int i = tid + k * WLF_THREADS;
          if (i < nv) r[k] = __ldcg(&p.rank_pack[r[k]]);
        }
#pragma unroll
        for (int k = 0; k < WLF_VPT; ++k) {
          const int i = tid + k * WLF_THREADS;
          if (i < nv) {
            const int id = s_prefix[r[k] >> WLF_RANK_BITS] + (r[k] & ((1 << WLF_RANK_BITS) - 1));
            lab_out[v0 + i] = id;
            lab_s[i] = id;
          }
        }
        __syncthreads();
        wlf_emit(p, v0, nv, lab_s, agg, level_base, (size_t)lv * V + v0, s_warp, mx, n_new, p.single);
      }
      if (b == 0 && tid == 0) {
        p.sc->level_dims[lv] = total;
        p.sc->level_base[lv + 1] = level_base + total;
      }
      level_base += total;
      flush_partials(lv);  // ends with __syncthreads: labels of this level are complete for the CTA's graphs
      WLF_STAMP(lv, 6);
    }
  }
}

}  // namespace gk
