// All WL levels in ONE persistent cooperative kernel (weisfeiler_lehman.py:199-258 + vertex_histogram.py:107-122 for
// every level), staged through shared memory.
//
// Why: the multi-kernel pipeline of wl.cuh spends each level in five latency-bound launches, far above its HBM floor.
// Micro-benchmarks (tools/mb/wl_mb.cu) show the limit is the number of SCATTERED L2 operations per vertex, so this
// kernel is organised to minimise them:
//
//   * The graphs are cut into TILES of whole graphs (<= WLF_TILE_V vertices, <= WLF_TILE_E edges); each CTA owns a
//     contiguous run of tiles.  A tile's CSR slice and labels are staged into shared memory with coalesced loads;
//     neighbour gathers, sorting and the per-graph label counts never leave shared memory.
//   * Signature dedup: the hash proposes, the signature verifies.  ONE packed 64-bit word per slot, {tag | single |
//     representative vertex}: insert = one CAS, plus one atomicMin when a further member of the class has to clear
//     the single bit or bring a smaller representative.
//   * (graph, column) counts are produced inside the graph in shared memory (a graph never straddles a tile) and
//     written to a compact COO list: no global feature hash table to fill and clear per level.
//   * The compressed label of a class is the id of its REPRESENTATIVE vertex (the smallest vertex of the class),
//     not a dense rank.  The reference's ids never leave the estimator (SURVEY 7: "bit-exact integer labels" =
//     identical label partition), and K only needs distinct columns per class.  So a level needs no CTA-local ranks,
//     no scan of the CTA counts and no rank gather, and ONE grid barrier: a level is   [A] signatures + insert | grid
//     barrier | [B] representative, verification, labels, feature entries.   Level l >= 1 owns the column range
//     [n_labels0 + (l-1) V, n_labels0 + l V).
//     Dense first-occurrence ids (gk_wl_labels, the WL-SP base kernel) are produced on demand by wl_densify.
//   * A vertex whose class has a single member in the whole data set is FROZEN: its label (= its own id) never
//     changes again, it needs no signature, insert or verification at deeper levels, and its feature column
//     occurs in one graph only, i.e. it contributes 1 to its graph's self similarity per remaining level and
//     nothing else.  That contribution is added once, when the vertex freezes, and no feature entry is ever
//     written for it.  At BASELINE config 2, 93 % of the vertices freeze at level 2 and 96 % by level 3: levels
//     3..5 touch 4 % of the data.
//   * Three signature tables rotate (level l uses table l mod 3; the table of level l+2 is cleared in [B] of
//     level l) and the verification rows are double-buffered by level parity, which is what makes the single
//     barrier sufficient: a CTA that is already in [A] of level l+1 never touches what a CTA still in [B] of
//     level l reads (a CTA cannot be two levels ahead: the barrier of l+1 waits for everybody's [B] of l).
//   * A CTA that owns one tile keeps its CSR slice, labels and frozen flags resident in shared memory across
//     levels.
//
// Exactness: every non-frozen vertex's full signature (own label, degree, sorted neighbour labels)
// is compared with its representative's; a mismatch raises the collision flag and the host retries with a new seed.
#pragma once
#include "common.cuh"
#include "wl.cuh"

namespace gk {

constexpr int WLF_THREADS = 1024;
constexpr int WLF_TILE_V = 4096;    // vertices per tile (u16 local indices)
constexpr int WLF_TILE_E = 16384;   // edges per tile
constexpr int WLF_VPT = WLF_TILE_V / WLF_THREADS;  // vertices per thread and tile (register batches)
constexpr int WLF_AGG = 8192;       // per-tile column -> graph-count aggregation table (shared memory)
static_assert(WLF_AGG * 8 <= WLF_TILE_E * 4, "aggregation table must fit in the sig_s region");
constexpr int WLF_CTA_V_LIMIT = 1 << 20;  // vertices per CTA: an input whose tiles give a CTA this many or more takes
                                          // the per-level kernels (wl.cuh)

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

struct WlFused2Params {
  int V, L;
  int n_labels0;
  const int* graph_ptr;
  const int* row_ptr;
  const int* col_idx;
  const int* vgraph;
  const int* labels0;
  const int* tile_vbeg;  // [n_tiles + 1] first vertex of each tile (whole graphs)
  const int* cta_tile;   // [grid + 1] first tile of each CTA
  int* labels_all;       // [L * V]; level 0: the packed dense ids, level >= 1: representative vertex ids
  int* sig_nbr;          // [2][E] sorted neighbour labels of the non-frozen vertices, double-buffered by level parity:
                         // with one barrier per level a fast CTA writes the rows of level l+1 while a slow one still
                         // verifies against the rows of level l
  long long E;
  int* slot_of;          // [V] hash slot of the vertex's signature at the current level (bit 31: the vertex installed the slot)
  int* payload;          // [2][ht_cap][8] the installing vertex's signature next to its slot, double-buffered by level
                         // parity like sig_nbr; NULL = verify against the representative's CSR row (first scheme)
  unsigned char* frozen; // [V] zeroed by the host
  unsigned long long* table;  // 3 x (ht_mask + 1) packed {31-bit tag | single | representative}; table 1 cleared by the host
  unsigned ht_mask;
  unsigned long long* coo_keys;  // feature entries: graph << 32 | column; fixed region of nv slots per (tile, level)
  unsigned* coo_cnt;
  unsigned* barrier;  // zeroed by the host before the launch
  unsigned long long seed;
  int degen_from;     // levels >= degen_from hash (own label, degree) only (gk_selftest_wl_collision); INT_MAX = off
  FeatStats st;
  unsigned long long* diag_frozen;  // [N] zeroed by the host: the frozen vertices' share of st.diag (WL-OA re-adds it)
  DevScalars* sc;     // level_dims[1..] zeroed by the host, level_base[0], [1] set
  long long* prof;    // optional [grid][L][16] globaltimer stamps (GRAKEL_B200_PROF), else NULL
};

// Feature entries of one tile from the labels in lab_s: a non-frozen vertex i emits (graph, base + label, count)
// iff it is the first vertex of its graph carrying that label; frozen vertices (unique labels) emit nothing.
// Fixed COO region per (tile, level), unused slots hold EMPTY64; per-column graph counts go through a shared-memory
// aggregation table first (a column shared by every graph costs one global atomic per tile).
// Per-vertex label multiplicity inside its graph and ONE emitting vertex per (graph, label):
// cf_s[i] = count | (emitter ? 0x8000 : 0) for the non-frozen vertices.
//   dense tiles (levels 0-2: most vertices still active): a shared-memory hash table keyed by (graph, label) -- the
//     slot word is {count : 16 | tile index of the vertex that installed it : 16}, the key is compared through that
//     vertex -- so every vertex costs one probe sequence and one atomic instead of a scan of its whole graph
//     (a scan of the whole graph per vertex was the costliest phase of the dense levels);
//   sparse tiles (deep levels: a few per cent active): the active vertices are compacted and each one is handled by a
//     whole warp whose lanes scan the graph in parallel (ballot + popc).
constexpr int WLF2_CT = 8192;  // slots of the (graph, label) table: >= 2 x WLF_TILE_V
static_assert(WLF2_CT >= 2 * WLF_TILE_V && WLF2_CT * 4 <= WLF_TILE_V * 8, "the table lives in the key_s region");
__device__ __forceinline__ void wlf2_count(const WlFused2Params& p, int nv, const int* lab_s, const unsigned char* frz_s,
                                           const int* gid_s, const unsigned short* gbeg_s, const unsigned short* gend_s,
                                           unsigned short* cf_s, unsigned* ct, unsigned short* list_s, int* s_warp) {
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  int mine = 0;
#pragma unroll
  for (int k = 0; k < WLF_VPT; ++k) {
    const int i = tid + k * WLF_THREADS;
    mine += (i < nv && !frz_s[i]) ? 1 : 0;
  }
  int n_act;
  const int ex0 = wlf_block_scan(mine, &n_act, s_warp);
  if (4 * n_act > nv) {
    for (int s2 = tid; s2 < WLF2_CT; s2 += WLF_THREADS) ct[s2] = 0xFFFFFFFFu;
    __syncthreads();
    // the installing vertex keeps its slot in cf_s (emitter bit | slot) until every vertex has counted
#pragma unroll
    for (int k = 0; k < WLF_VPT; ++k) {
      const int i = tid + k * WLF_THREADS;
      if (i < nv && !frz_s[i]) {
        cf_s[i] = 0;
        const int l = lab_s[i], g = gid_s[i];
        unsigned h = (((unsigned)l * 0x9E3779B1u) ^ ((unsigned)g * 0x85EBCA77u)) >> 15 & (WLF2_CT - 1);
        while (true) {
          unsigned w = ct[h];
          if (w == 0xFFFFFFFFu) {
            w = atomicCAS(&ct[h], 0xFFFFFFFFu, (1u << 16) | (unsigned)i);
            if (w == 0xFFFFFFFFu) { cf_s[i] = (unsigned short)(0x8000u | h); break; }
          }
          const unsigned o = w & 0xFFFFu;
          if (lab_s[o] == l && gid_s[o] == g) { atomicAdd(&ct[h], 1u << 16); break; }
          h = (h + 1) & (WLF2_CT - 1);
        }
      }
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < WLF_VPT; ++k) {
      const int i = tid + k * WLF_THREADS;
      if (i < nv && !frz_s[i] && (cf_s[i] & 0x8000u)) cf_s[i] = (unsigned short)((ct[cf_s[i] & 0x7FFFu] >> 16) | 0x8000u);
    }
  } else {
    int ex = ex0;
#pragma unroll
    for (int k = 0; k < WLF_VPT; ++k) {
      const int i = tid + k * WLF_THREADS;
      if (i < nv && !frz_s[i]) list_s[ex++] = (unsigned short)i;
    }
    __syncthreads();
    for (int a = wid; a < n_act; a += WLF_THREADS / 32) {
      const int i = list_s[a];
      const int gs = gbeg_s[i], ge = gend_s[i], l = lab_s[i];
      int cnt = 0;
      bool earlier = false;
      for (int u0 = gs; u0 < ge; u0 += 32) {
        const int u = u0 + lane;
        const bool same = u < ge && lab_s[u] == l;
        const unsigned m = __ballot_sync(0xffffffffu, same);
        cnt += __popc(m);
        earlier = earlier || (__ballot_sync(0xffffffffu, same && u < i) != 0u);
      }
      if (lane == 0) cf_s[i] = (unsigned short)(cnt | (earlier ? 0 : 0x8000));
    }
  }
}

__device__ __forceinline__ void wlf2_emit(const WlFused2Params& p, int v0, int nv, const int* lab_s, const unsigned char* frz_s,
                                          const int* gid_s, const unsigned short* gbeg_s, const unsigned short* gend_s,
                                          unsigned short* cf_s, unsigned* ct, unsigned short* list_s,
                                          unsigned* agg, long long base, size_t coo_off, int* s_warp, unsigned& mx, unsigned& n_new) {
  const int tid = threadIdx.x, lane = tid & 31;
  wlf2_count(p, nv, lab_s, frz_s, gid_s, gbeg_s, gend_s, cf_s, ct, list_s, s_warp);
  __syncthreads();
  // a vertex emits iff it is not frozen and carries the emitter bit; read again from shared memory below rather than
  // kept in registers across the scan
  int n_emit = 0;
#pragma unroll
  for (int k = 0; k < WLF_VPT; ++k) {
    const int i = tid + k * WLF_THREADS;
    n_emit += (i < nv && !frz_s[i] && (cf_s[i] & 0x8000u)) ? 1 : 0;
  }
  int total;
  int ex = wlf_block_scan(n_emit, &total, s_warp);
  // few entries (deep levels, where most vertices are frozen): straight to the global column counters; otherwise
  // aggregate per tile in shared memory first (a column shared by every graph costs one global atomic per tile)
  const bool use_agg = total > 256;
  if (use_agg) {
    for (int s = tid; s < WLF_AGG * 2; s += WLF_THREADS) agg[s] = (s & 1) ? 0u : 0xFFFFFFFFu;  // {column, graphs}
    __syncthreads();
  }
  for (int i = total + tid; i < nv; i += WLF_THREADS) p.coo_keys[coo_off + i] = EMPTY64;  // unused rest of the fixed region
#pragma unroll
  for (int k = 0; k < WLF_VPT; ++k) {
    const int i = tid + k * WLF_THREADS;
    const int gg = i < nv ? gid_s[i] : -1;  // every vertex of the tile, frozen or not: graphs stay contiguous lane runs
    const unsigned cf = (i < nv && !frz_s[i]) ? cf_s[i] : 0u;
    const bool emit = (cf & 0x8000u) != 0;
    const unsigned cnt = cf & 0x7FFFu;
    if (emit) {
      const unsigned col = (unsigned)(base + lab_s[i]);
      p.coo_keys[coo_off + ex] = ((unsigned long long)(unsigned)gg << 32) | col;
      p.coo_cnt[coo_off + ex] = cnt;
      ++ex;
      mx = max(mx, cnt);
      n_new += 1u;
      if (use_agg) {
        unsigned slot = (col * 0x9E3779B1u >> 12) & (WLF_AGG - 1);
        while (true) {
          unsigned prev = agg[2 * slot];
          if (prev == 0xFFFFFFFFu) prev = atomicCAS(&agg[2 * slot], 0xFFFFFFFFu, col);
          if (prev == 0xFFFFFFFFu || prev == col) { atomicAdd(&agg[2 * slot + 1], 1u); break; }
          slot = (slot + 1) & (WLF_AGG - 1);
        }
      } else {
        atomicAdd(&p.st.colcnt[col], 1u);
      }
    }
    // exact self similarity: sum of squared counts per graph (runs of equal g inside the warp)
    unsigned long long val = emit ? (unsigned long long)cnt * cnt : 0ULL;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const unsigned long long y = __shfl_down_sync(0xffffffffu, val, d);
      const int gy = __shfl_down_sync(0xffffffffu, gg, d);
      if (lane + d < 32 && gy == gg) val += y;
    }
    const int gprev = __shfl_up_sync(0xffffffffu, gg, 1);
    if (gg >= 0 && (lane == 0 || gprev != gg) && val) atomicAdd(&p.st.diag[gg], val);
  }
  if (use_agg) {
    __syncthreads();
    for (int s = tid; s < WLF_AGG; s += WLF_THREADS) {
      const unsigned col = agg[2 * s];
      if (col != 0xFFFFFFFFu) atomicAdd(&p.st.colcnt[col], agg[2 * s + 1]);
    }
  }
  __syncthreads();  // agg is reused by the next tile / overwritten by the next level's signatures
}

// The tile's non-frozen vertices in ascending order, act_s[0, n_act).  [A], [B] and the label write-back of a level
// run over this list, so the deep levels (a few per cent of the vertices still active) cost their live vertices, not
// the tile.  Ascending, so the vertices of one graph stay contiguous lane runs ([B]'s per-graph sums).
__device__ __forceinline__ int wlf2_compact(int nv, const unsigned char* frz_s, unsigned short* act_s, int* s_warp) {
  const int i0 = threadIdx.x * WLF_VPT;
  int mine = 0;
#pragma unroll
  for (int k = 0; k < WLF_VPT; ++k) mine += (i0 + k < nv && !frz_s[i0 + k]) ? 1 : 0;
  int n_act;
  int ex = wlf_block_scan(mine, &n_act, s_warp);
#pragma unroll
  for (int k = 0; k < WLF_VPT; ++k)
    if (i0 + k < nv && !frz_s[i0 + k]) act_s[ex++] = (unsigned short)(i0 + k);
  __syncthreads();
  return n_act;
}

constexpr int WLF2_SMEM = (WLF_TILE_V + 2) * 4 /*rp_s*/ + WLF_TILE_V * 8 /*key_s | ct*/ + WLF_TILE_V * 4 /*lab_s*/ +
                          WLF_TILE_E * 4 /*sig_s | agg*/ + WLF_TILE_E * 2 /*col_s*/ + WLF_TILE_V /*frz_s*/ +
                          WLF_TILE_V * 4 /*gid_s*/ + WLF_TILE_V * 4 /*gbeg_s, gend_s*/ + WLF_TILE_V * 4 /*slot_s | list_s*/ +
                          WLF_TILE_V * 2 /*cf_s | act_s*/ + 16;
static_assert(WLF2_SMEM <= 232448, "shared memory budget of one CTA");

// Global -> shared staging of a tile with several loads in flight per thread.  A plain strided loop keeps ONE load
// per thread outstanding: 1024 threads x 4 bytes per ~1 us of L2 latency is ~4 GB/s per SM, and a CTA that owns more
// than one tile (V > SMs x 4096) would re-stage ~100 KB per tile, level and phase that way, which dominates the kernel
// at the multi-GPU sizes.
#define WLF2_STAGE4(N_, LOAD_, STORE_)                                                     \
  for (int i0_ = tid; i0_ < (N_); i0_ += 4 * WLF_THREADS) {                                 \
    const int i1_ = i0_ + WLF_THREADS, i2_ = i0_ + 2 * WLF_THREADS, i3_ = i0_ + 3 * WLF_THREADS; \
    const int x0_ = LOAD_(i0_);                                                              \
    const int x1_ = i1_ < (N_) ? LOAD_(i1_) : 0;                                             \
    const int x2_ = i2_ < (N_) ? LOAD_(i2_) : 0;                                             \
    const int x3_ = i3_ < (N_) ? LOAD_(i3_) : 0;                                             \
    STORE_(i0_, x0_);                                                                        \
    if (i1_ < (N_)) STORE_(i1_, x1_);                                                        \
    if (i2_ < (N_)) STORE_(i2_, x2_);                                                        \
    if (i3_ < (N_)) STORE_(i3_, x3_);                                                        \
  }
__device__ __forceinline__ void wlf2_stage_csr(const WlFused2Params& p, int v0, int nv, int e0, int ne, int* rp_s,
                                               unsigned short* col_s, int tid) {
#define LD_(i) p.row_ptr[v0 + (i)]
#define ST_(i, x) rp_s[(i)] = (x) - e0
  WLF2_STAGE4(nv + 1, LD_, ST_)
#undef LD_
#undef ST_
#define LD_(k) p.col_idx[e0 + (k)]
#define ST_(k, x) col_s[(k)] = (unsigned short)((x) - v0)
  WLF2_STAGE4(ne, LD_, ST_)
#undef LD_
#undef ST_
}
__device__ __forceinline__ void wlf2_stage_labels(const WlFused2Params& p, const int* lab_in, int v0, int nv, int* lab_s,
                                                  unsigned char* frz_s, int tid) {
#define LD_(i) lab_in[v0 + (i)]
#define ST_(i, x) lab_s[(i)] = (x)
  WLF2_STAGE4(nv, LD_, ST_)
#undef LD_
#undef ST_
#define LD_(i) (int)p.frozen[v0 + (i)]
#define ST_(i, x) frz_s[(i)] = (unsigned char)(x)
  WLF2_STAGE4(nv, LD_, ST_)
#undef LD_
#undef ST_
}

// PAY: slot payloads (see [A3]) instead of the representative's CSR row as the verification reference.  A template
// parameter, not a runtime switch: with both schemes live in one instance the kernel spilled 368 bytes per thread
// at its 64-register budget.  Compiled for sm_90a, each instance alone fits the 64 registers with no spill (ptxas
// -v: 0 bytes of spill stores and loads) because no phase holds more than a pair of items in registers ([A3], [B]),
// the feature phase re-reads its per-vertex state from shared memory, and one warp reduces the per-CTA partials.
template <bool PAY>
__global__ void __launch_bounds__(WLF_THREADS, 1)
wl_fused2_kernel(WlFused2Params p) {
  extern __shared__ __align__(16) unsigned char wlf_smem[];
  int* rp_s = reinterpret_cast<int*>(wlf_smem);
  unsigned long long* key_s = reinterpret_cast<unsigned long long*>(rp_s + (WLF_TILE_V + 2));
  int* lab_s = reinterpret_cast<int*>(key_s + WLF_TILE_V);
  int* sig_s = lab_s + WLF_TILE_V;
  unsigned* agg = reinterpret_cast<unsigned*>(sig_s);  // emit phase only
  unsigned short* col_s = reinterpret_cast<unsigned short*>(sig_s + WLF_TILE_E);
  unsigned char* frz_s = reinterpret_cast<unsigned char*>(col_s + WLF_TILE_E);
  int* gid_s = reinterpret_cast<int*>(frz_s + WLF_TILE_V);  // graph of every tile vertex
  unsigned short* gbeg_s = reinterpret_cast<unsigned short*>(gid_s + WLF_TILE_V);  // its graph's vertex range, tile-local
  unsigned short* gend_s = gbeg_s + WLF_TILE_V;
  // payload scheme, resident tiles: slot (| installer bit) of every tile vertex from [A] to [B] of a level; the same
  // region holds the emit phase's compaction list (list_s), which runs after [B] has consumed the slots
  unsigned* slot_s = reinterpret_cast<unsigned*>(gend_s + WLF_TILE_V);
  unsigned short* list_s = reinterpret_cast<unsigned short*>(slot_s);
  unsigned short* cf_s = reinterpret_cast<unsigned short*>(slot_s + WLF_TILE_V);  // emit phase: in-graph count | emitter bit
  unsigned short* act_s = cf_s;  // [A] to the label write-back: the tile's non-frozen vertices (wlf2_compact)
  unsigned* ct = reinterpret_cast<unsigned*>(key_s);  // emit phase: the (graph, label) table (key_s is free after [A])
  __shared__ int s_warp[32];
  __shared__ unsigned s_red[128];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int G = gridDim.x, b = blockIdx.x;
  const int t_beg = p.cta_tile[b], t_end = p.cta_tile[b + 1];
  const bool resident = (t_end - t_beg) == 1;  // one tile: CSR slice, labels, frozen flags stay in shared memory
  const int V = p.V;
  const size_t ht_cap = (size_t)p.ht_mask + 1;
  unsigned n_sync = 0;
  unsigned mx = 0, n_new = 0, n_rep = 0, n_fz = 0;  // n_fz: self-similarity units of vertices frozen at this level
  WLF_STAMP(0, 0);

  // publish the per-CTA partials of a level (max count, created entries) and add the CTA's class count
  auto flush_partials = [&](int level) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
      mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, d));
      n_new += __shfl_xor_sync(0xffffffffu, n_new, d);
      n_rep += __shfl_xor_sync(0xffffffffu, n_rep, d);
      n_fz += __shfl_xor_sync(0xffffffffu, n_fz, d);
    }
    if (lane == 0) { s_red[wid] = mx; s_red[32 + wid] = n_new; s_red[64 + wid] = n_rep; s_red[96 + wid] = n_fz; }
    __syncthreads();
    if (wid == 0) {  // one warp reduces the 32 warp partials (one thread unrolling it was the kernel's register peak)
      unsigned m = s_red[lane], n = s_red[32 + lane], r = s_red[64 + lane], z = s_red[96 + lane];
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) {
        m = max(m, __shfl_xor_sync(0xffffffffu, m, d));
        n += __shfl_xor_sync(0xffffffffu, n, d);
        r += __shfl_xor_sync(0xffffffffu, r, d);
        z += __shfl_xor_sync(0xffffffffu, z, d);
      }
      if (lane == 0) {
        if (z) atomicAdd(&p.sc->sp_coo, (unsigned long long)z);  // total of diag_frozen (WL-OA's entry count)
        p.st.part_max[(size_t)level * G + b] = m;
        p.st.part_new[(size_t)level * G + b] = n;
        if (level > 0 && r) atomicAdd((unsigned long long*)&p.sc->level_dims[level], (unsigned long long)r);
      }
    }
    mx = 0; n_new = 0; n_rep = 0; n_fz = 0;
    __syncthreads();
  };

  auto stage_graphs = [&](int v0, int nv) {
#define LD_(i) p.vgraph[v0 + (i)]
#define ST_(i, x) gid_s[(i)] = (x)
    WLF2_STAGE4(nv, LD_, ST_)
#undef LD_
#undef ST_
    // (each thread re-reads what it wrote itself: same index mapping, no barrier needed)
#define LD_(i) p.graph_ptr[gid_s[(i)]]
#define ST_(i, x) gbeg_s[(i)] = (unsigned short)((x) - v0)
    WLF2_STAGE4(nv, LD_, ST_)
#undef LD_
#undef ST_
#define LD_(i) p.graph_ptr[gid_s[(i)] + 1]
#define ST_(i, x) gend_s[(i)] = (unsigned short)((x) - v0)
    WLF2_STAGE4(nv, LD_, ST_)
#undef LD_
#undef ST_
  };

  // ---- level 0: labels as given (dense ids); nothing is frozen yet
  for (int t = t_beg; t < t_end; ++t) {
    const int v0 = p.tile_vbeg[t], nv = p.tile_vbeg[t + 1] - v0;
    __syncthreads();
#define LD_(i) p.labels0[v0 + (i)]
#define ST_(i, x) { lab_s[(i)] = (x); p.labels_all[v0 + (i)] = (x); frz_s[(i)] = 0; }
    WLF2_STAGE4(nv, LD_, ST_)
#undef LD_
#undef ST_
    stage_graphs(v0, nv);
    if (resident) {  // stage the CSR slice once
      const int e0 = p.row_ptr[v0], ne = p.row_ptr[v0 + nv] - e0;
      wlf2_stage_csr(p, v0, nv, e0, ne, rp_s, col_s, tid);
    }
    __syncthreads();
    WLF_STAMP(0, 1);
    wlf2_emit(p, v0, nv, lab_s, frz_s, gid_s, gbeg_s, gend_s, cf_s, ct, list_s, agg, 0, (size_t)v0, s_warp, mx, n_new);
    WLF_STAMP(0, 2);
  }
  if (p.L > 2) {  // table of level 2 (first touched after the barrier of level 1)
    const uint4 ones = make_uint4(0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu);
    uint4* hk = reinterpret_cast<uint4*>(p.table + 2 * ht_cap);
    for (size_t i = (size_t)b * WLF_THREADS + tid; i < ht_cap / 2; i += (size_t)G * WLF_THREADS) hk[i] = ones;
  }
  if (b == 0 && tid == 0)
    for (int lv = 1; lv < p.L; ++lv) p.sc->level_base[lv + 1] = (long long)p.n_labels0 + (long long)lv * V;
  WLF_STAMP(0, 3);
  flush_partials(0);
  WLF_STAMP(0, 6);

  for (int lv = 1; lv < p.L; ++lv) {
    const int* lab_in = p.labels_all + (size_t)(lv - 1) * V;
    int* lab_out = p.labels_all + (size_t)lv * V;
    unsigned long long* tab = p.table + (size_t)(lv % 3) * ht_cap;
    const long long level_base = (long long)p.n_labels0 + (long long)(lv - 1) * V;
    int* sig_g = p.sig_nbr + (size_t)(lv & 1) * (size_t)p.E;  // this level's rows
    int* pay = PAY ? p.payload + (size_t)(lv & 1) * ht_cap * 8 : nullptr;  // this level's slot payloads

    // ---------------- [A] signatures + insert (non-frozen vertices)
    WLF_STAMP(lv, 0);
    int n_act = 0;  // resident tile: the list built in [A] serves [B] of the same level
    for (int t = t_beg; t < t_end; ++t) {
      const int v0 = p.tile_vbeg[t], nv = p.tile_vbeg[t + 1] - v0;
      const int e0 = p.row_ptr[v0], ne = p.row_ptr[v0 + nv] - e0;
      if (!resident) {
        __syncthreads();  // previous tile's shared memory is no longer read
        wlf2_stage_csr(p, v0, nv, e0, ne, rp_s, col_s, tid);
        wlf2_stage_labels(p, lab_in, v0, nv, lab_s, frz_s, tid);
        __syncthreads();
      }
      n_act = wlf2_compact(nv, frz_s, act_s, s_warp);
      WLF_STAMP(lv, 8);
      // [A1] one thread per vertex of degree <= 8: 19-comparator network in registers
      for (int a = tid; a < n_act; a += WLF_THREADS) {
        const int i = act_s[a];
        const int beg = rp_s[i];
        const int deg = rp_s[i + 1] - beg;
        if (deg > 8) continue;
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
      // [A2] higher degrees: one warp per vertex (shuffle bitonic <= 32, in-segment bitonic above)
      for (int a0 = wid * 32; a0 < n_act; a0 += WLF_THREADS) {
        const int iv = a0 + lane < n_act ? act_s[a0 + lane] : 0;
        const bool big = a0 + lane < n_act && (rp_s[iv + 1] - rp_s[iv]) > 8;
        unsigned m = __ballot_sync(0xffffffffu, big);
        while (m) {
          const int i = __shfl_sync(0xffffffffu, iv, __ffs(m) - 1);
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
      // [A3] insert every non-frozen vertex of the tile.  Items in pairs, like [B]: the probes of two items are issued
      // together; item u of pair k0 is act_s[tid + (k0 + u) * WLF_THREADS], its tile index re-read from shared memory.
#pragma unroll 1
      for (int k0 = 0; k0 < WLF_VPT; k0 += 2) {
        if (tid + k0 * WLF_THREADS >= n_act) break;
        unsigned long long key[2], w[2];
        unsigned slot[2];
        bool act[2], won[2];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int a = tid + (k0 + u) * WLF_THREADS;
          act[u] = a < n_act;
          key[u] = act[u] ? key_s[act_s[a]] : 0ULL;
          won[u] = false;
          slot[u] = (unsigned)((key[u] & 0xFFFFFFFFULL) * 0x9E3779B1ULL >> 8) & p.ht_mask;
        }
        bool any = true;
        while (any) {
          // CAS first (no read-before-CAS): a new signature costs ONE L2 round trip; an existing one gets the
          // slot's word back from the failed CAS
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            if (!act[u]) { w[u] = 0ULL; continue; }
            const unsigned long long mine = (key[u] & 0xFFFFFFFE00000000ULL) | (1ULL << 32) |
                                            (unsigned)(v0 + act_s[tid + (k0 + u) * WLF_THREADS]);
            w[u] = atomicCAS(&tab[slot[u]], EMPTY64, mine);
          }
          any = false;
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            if (!act[u]) continue;
            if (w[u] == EMPTY64) { act[u] = false; won[u] = true; continue; }  // the CAS installed our word (single bit set)
            if ((w[u] >> 33) == (key[u] >> 33)) {
              const unsigned rep = (unsigned)w[u];
              const unsigned v = (unsigned)(v0 + act_s[tid + (k0 + u) * WLF_THREADS]);
              // a second member: clear the single bit and keep the smaller representative in one atomicMin
              if (((w[u] >> 32) & 1ULL) || rep > v)
                atomicMin(&tab[slot[u]], (key[u] & 0xFFFFFFFE00000000ULL) | min(rep, v));
              act[u] = false;
              continue;
            }
            slot[u] = (slot[u] + 1) & p.ht_mask;
            any = true;
          }
        }
        if (PAY) {
          // Verification data travels WITH the slot: the vertex whose CAS installed a slot writes its full signature
          // {label, degree, first sorted neighbour labels} into the slot's 32-byte payload; every other vertex that
          // matched the slot's tag compares its own signature with that payload in [B] -- one L2 round trip next to the
          // table word instead of the chain slot -> representative -> CSR row -> neighbour row.  Sound: all vertices
          // of a slot that pass carry the installer's signature, i.e. they are one class; any other vertex raises the
          // collision flag.  Degrees above 6: the payload holds five labels and the installer's row offset, the rest of
          // the row is compared through sig_nbr (only installers of such degrees write their rows there).
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            const int a = tid + (k0 + u) * WLF_THREADS;
            if (a >= n_act) continue;
            const int i = act_s[a];
            const unsigned sw = slot[u] | (won[u] ? 0x80000000u : 0u);
            if (resident) slot_s[i] = sw; else p.slot_of[v0 + i] = (int)sw;
            if (won[u]) {
              const int beg = rp_s[i], deg = rp_s[i + 1] - beg;
              int nb[6];
#pragma unroll
              for (int j = 0; j < 6; ++j) nb[j] = j < deg ? sig_s[beg + j] : 0x7fffffff;
              if (deg > 6) nb[5] = e0 + beg;
              uint4* dst = reinterpret_cast<uint4*>(pay + (size_t)slot[u] * 8);
              dst[0] = make_uint4((unsigned)lab_s[i], (unsigned)deg, (unsigned)nb[0], (unsigned)nb[1]);
              dst[1] = make_uint4((unsigned)nb[2], (unsigned)nb[3], (unsigned)nb[4], (unsigned)nb[5]);
              if (resident && deg > 6)
                for (int j = 5; j < deg; ++j) sig_g[e0 + beg + j] = sig_s[beg + j];
            }
          }
        } else {
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            const int a = tid + (k0 + u) * WLF_THREADS;
            if (a < n_act) p.slot_of[v0 + act_s[a]] = (int)slot[u];
          }
        }
      }
      // sorted neighbour labels of the inserted vertices to global memory: other CTAs verify against them.  Most of
      // the tile inserting: one coalesced copy of the whole segment array (stale rows are never read); few: row by row
      // (payload scheme on a resident tile: nothing -- own rows stay in shared memory, see above)
      if (PAY && resident) {
      } else if (2 * n_act >= nv) {
        for (int j = tid; j < ne; j += WLF_THREADS) sig_g[e0 + j] = sig_s[j];
      } else {
        for (int a = tid; a < n_act; a += WLF_THREADS) {
          const int i = act_s[a];
          const int beg = rp_s[i], end = rp_s[i + 1];
          for (int j = beg; j < end; ++j) sig_g[e0 + j] = sig_s[j];
        }
      }
    }
    __syncthreads();
    WLF_STAMP(lv, 1);
    wlf_grid_sync(p.barrier, (++n_sync) * (unsigned)G);
    WLF_STAMP(lv, 2);

    // ---------------- [B] representative, verification, new labels, freezing, feature entries
    for (int t = t_beg; t < t_end; ++t) {
      const int v0 = p.tile_vbeg[t], nv = p.tile_vbeg[t + 1] - v0;
      if (!resident) {
        __syncthreads();
        wlf2_stage_labels(p, lab_in, v0, nv, lab_s, frz_s, tid);
        stage_graphs(v0, nv);
        __syncthreads();
        n_act = wlf2_compact(nv, frz_s, act_s, s_warp);
      }
      if (tid == 0) n_rep += (unsigned)(nv - n_act);  // a frozen vertex is a class of its own at every level
      int* res_s = reinterpret_cast<int*>(key_s);  // per list position: new label | 0x80000000 if it freezes now
      // Items in pairs: the table words and payloads of two items are in flight together, and nothing of a pair stays
      // live in registers past it (under the 64-register budget of 1024 threads the whole batch of four spilled).
#pragma unroll 1
      for (int k0 = 0; k0 < WLF_VPT; k0 += 2) {
        if ((tid & ~31) + k0 * WLF_THREADS >= n_act) break;  // warp-uniform: no item of this warp from here on
        unsigned long long word[2];
        uint4 pl0[2], pl1[2];  // payload scheme: the installer's signature (vertices that did not install)
        bool chk[2];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int a = tid + (k0 + u) * WLF_THREADS;
          word[u] = 0ULL;
          chk[u] = false;
          pl0[u] = pl1[u] = make_uint4(0u, 0u, 0u, 0u);
          if (a < n_act) {
            const int i = act_s[a];
            const unsigned sw = (PAY && resident) ? slot_s[i] : (unsigned)p.slot_of[v0 + i];
            const unsigned sl = PAY ? sw & 0x7fffffffu : sw;
            if (PAY && !(sw >> 31)) {
              chk[u] = true;
              const uint4* src = reinterpret_cast<const uint4*>(pay + (size_t)sl * 8);
              pl0[u] = __ldcg(src);
              pl1[u] = __ldcg(src + 1);
            }
            word[u] = __ldcg(&tab[sl]);
          }
        }
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int a = tid + (k0 + u) * WLF_THREADS;
          const bool act = a < n_act;
          const int i = act ? act_s[a] : 0;
          const int v = v0 + i;
          const int r = (int)(unsigned)word[u];
          const bool sgl = act && ((word[u] >> 32) & 1ULL) && r == v;
          unsigned long long fz = 0ULL;  // self-similarity contribution of a vertex that freezes now
          const int gg = act ? gid_s[i] : -1;
          if (act) {
            // verification against the representative: CSR row and label of both sides, then the sorted labels
            if (PAY) {
              if (chk[u]) {  // compare with the installer's signature in the slot payload
                int bv, d;
                if (resident) { bv = rp_s[i]; d = rp_s[i + 1] - bv; }
                else { bv = p.row_ptr[v]; d = p.row_ptr[v + 1] - bv; }
                const int pn[6] = {(int)pl0[u].z, (int)pl0[u].w, (int)pl1[u].x, (int)pl1[u].y, (int)pl1[u].z, (int)pl1[u].w};
                bool same = ((int)pl0[u].x == lab_s[i]) && ((int)pl0[u].y == d);
                if (same) {
                  const int nd = d > 6 ? 5 : d;
#pragma unroll
                  for (int j = 0; j < 6; ++j)
                    if (j < nd) same = same && ((resident ? sig_s[bv + j] : sig_g[bv + j]) == pn[j]);
                  if (d > 6) {
                    const int off = pn[5];  // installer's row offset in sig_nbr
                    for (int j = 5; same && j < d; ++j)
                      same = (resident ? sig_s[bv + j] : sig_g[bv + j]) == __ldcg(&sig_g[off + j]);
                  }
                }
                if (!same) atomicOr(&p.sc->collision, 1u << min(lv, 30));  // bit = level (error message / retry)
              }
              if (r == v) n_rep += 1u;
            } else if (r != v) {
              int bv, dv;
              if (resident) { bv = rp_s[i]; dv = rp_s[i + 1] - bv; }  // own side from shared memory (sig_s)
              else { bv = p.row_ptr[v]; dv = p.row_ptr[v + 1] - bv; }
              const int br = p.row_ptr[r], dr = p.row_ptr[r + 1] - br;
              bool same = (dv == dr) && (lab_s[i] == __ldcg(&lab_in[r]));
              if (same && dv <= 8) {
                int x[8], c[8];
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                  x[j] = j < dv ? (resident ? sig_s[bv + j] : sig_g[bv + j]) : 0;
                  c[j] = j < dv ? __ldcg(&sig_g[br + j]) : 0;
                }
#pragma unroll
                for (int j = 0; j < 8; ++j) same = same && (x[j] == c[j]);
              } else {
                for (int j = 0; same && j < dv; ++j)
                  same = (resident ? sig_s[bv + j] : sig_g[bv + j]) == __ldcg(&sig_g[br + j]);
              }
              if (!same) atomicOr(&p.sc->collision, 1u << min(lv, 30));  // bit = level (error message / retry)
            } else {
              n_rep += 1u;
            }
            if (sgl) {  // a class of one vertex: frozen from this level on, one diagonal unit per remaining level
              fz = (unsigned long long)(p.L - lv);
              n_new += (unsigned)(p.L - lv);
              n_fz += (unsigned)(p.L - lv);
              mx = max(mx, 1u);
            }
            res_s[a] = r | (sgl ? (int)0x80000000u : 0);
          }
          // per-graph aggregation of the frozen contributions (runs of equal graph inside the warp: the list ascends)
          unsigned long long val = fz;
#pragma unroll
          for (int d = 1; d < 32; d <<= 1) {
            const unsigned long long y = __shfl_down_sync(0xffffffffu, val, d);
            const int gy = __shfl_down_sync(0xffffffffu, gg, d);
            if (lane + d < 32 && gy == gg) val += y;
          }
          const int gprev = __shfl_up_sync(0xffffffffu, gg, 1);
          if (gg >= 0 && (lane == 0 || gprev != gg) && val) {
            atomicAdd(&p.st.diag[gg], val);
            atomicAdd(&p.diag_frozen[gg], val);
          }
        }
      }
      WLF_STAMP(lv, 4);
      __syncthreads();  // every thread has read the old labels of the tile it needs
      // new labels of the live vertices; a vertex that freezes writes its own id for every deeper level now, so a
      // frozen vertex is never visited again
      for (int a = tid; a < n_act; a += WLF_THREADS) {
        const int i = act_s[a], v = v0 + i, x = res_s[a], r = x & 0x7fffffff;
        lab_s[i] = r;
        lab_out[v] = r;
        if (x < 0) {
          frz_s[i] = 1;
          p.frozen[v] = 1;
          for (int l2 = lv + 1; l2 < p.L; ++l2) p.labels_all[(size_t)l2 * V + v] = v;
        }
      }
      __syncthreads();
      WLF_STAMP(lv, 5);
      wlf2_emit(p, v0, nv, lab_s, frz_s, gid_s, gbeg_s, gend_s, cf_s, ct, list_s, agg, level_base, (size_t)lv * V + v0, s_warp, mx, n_new);
    }
    WLF_STAMP(lv, 3);
    if (lv + 2 < p.L) {  // clear the table level lv+2 inserts into (last read in [B] of level lv-1, which every CTA has left)
      const uint4 ones = make_uint4(0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu);
      uint4* hk = reinterpret_cast<uint4*>(p.table + (size_t)((lv + 2) % 3) * ht_cap);
      for (size_t i = (size_t)b * WLF_THREADS + tid; i < ht_cap / 2; i += (size_t)G * WLF_THREADS) hk[i] = ones;
    }
    flush_partials(lv);  // ends with __syncthreads
    WLF_STAMP(lv, 6);
  }
}

// Everything the fused kernel expects to find cleared, in ONE launch (eight cudaMemsetAsync calls and a synchronous
// scalar upload cost more than the clears themselves): scalars, per-CTA partials, column counters, self
// similarities, the grid barrier, the frozen flags and the signature table of level 1.
struct Wlf2Prepare {
  DevScalars* sc; int n_labels0;
  unsigned* part_max; unsigned* part_new; long long n_part;
  unsigned* colcnt; long long col_cap;
  unsigned long long* diag; unsigned long long* diag_frozen; long long n_graphs;
  unsigned* barrier;
  unsigned char* frozen; long long V;
  unsigned long long* table1; long long ht_cap;
};
__global__ void __launch_bounds__(1024)
wlf2_prepare_kernel(Wlf2Prepare q) {
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x, nth = (long long)gridDim.x * blockDim.x;
  // scalars: all zero except level_dims[0] = level_base[1] = n_labels0 (what the host used to upload)
  if (tid < (long long)(sizeof(DevScalars) / 8)) {
    const bool is_n0 = tid == (long long)(offsetof(DevScalars, level_dims) / 8) ||
                       tid == (long long)(offsetof(DevScalars, level_base) / 8 + 1);
    reinterpret_cast<unsigned long long*>(q.sc)[tid] = is_n0 ? (unsigned long long)q.n_labels0 : 0ULL;
  }
  for (long long i = tid; i < q.n_part; i += nth) { q.part_max[i] = 0u; q.part_new[i] = 0u; }
  for (long long i = tid; i < q.n_graphs; i += nth) { q.diag[i] = 0ULL; q.diag_frozen[i] = 0ULL; }
  if (tid == 0) *q.barrier = 0u;
  {
    uint4* c4 = reinterpret_cast<uint4*>(q.colcnt);  // cudaMalloc'ed: 256-byte aligned
    const uint4 z = make_uint4(0u, 0u, 0u, 0u);
    for (long long i = tid; i < q.col_cap / 4; i += nth) c4[i] = z;
    for (long long i = q.col_cap / 4 * 4 + tid; i < q.col_cap; i += nth) q.colcnt[i] = 0u;
    uint4* f4 = reinterpret_cast<uint4*>(q.frozen);
    for (long long i = tid; i < q.V / 16; i += nth) f4[i] = z;
    for (long long i = q.V / 16 * 16 + tid; i < q.V; i += nth) q.frozen[i] = 0;
  }
  if (q.table1) {
    const uint4 ones = make_uint4(0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu);
    uint4* t4 = reinterpret_cast<uint4*>(q.table1);
    for (long long i = tid; i < q.ht_cap / 2; i += nth) t4[i] = ones;
  }
}
// ---- dense first-occurrence ids of one level >= 1 on demand (gk_wl_labels, WL-SP): representatives are the
// vertices with lab[v] == v; their rank in vertex order is the id the reference-order-free parity tests use.
constexpr int DENS_THREADS = 1024;
__global__ void __launch_bounds__(DENS_THREADS)
wl_dens_count(int V, const int* __restrict__ lab, int* __restrict__ block_sums) {
  __shared__ int s_warp[32];
  const int v = blockIdx.x * DENS_THREADS + threadIdx.x;
  const int f = (v < V && lab[v] == v) ? 1 : 0;
  int total;
  wlf_block_scan(f, &total, s_warp);
  if (threadIdx.x == 0) block_sums[blockIdx.x] = total;
}
__global__ void __launch_bounds__(DENS_THREADS)
wl_dens_scan(int nb, int* block_sums) {  // one block: exclusive scan in place
  __shared__ int s_warp[32];
  __shared__ int s_carry;
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  for (int i0 = 0; i0 < nb; i0 += DENS_THREADS) {
    const int i = i0 + threadIdx.x;
    const int x = i < nb ? block_sums[i] : 0;
    int total;
    const int ex = wlf_block_scan(x, &total, s_warp);
    if (i < nb) block_sums[i] = s_carry + ex;
    __syncthreads();
    if (threadIdx.x == 0) s_carry += total;
    __syncthreads();
  }
}
__global__ void __launch_bounds__(DENS_THREADS)
wl_dens_rank(int V, const int* __restrict__ lab, const int* __restrict__ block_sums, int* __restrict__ rank) {
  __shared__ int s_warp[32];
  const int v = blockIdx.x * DENS_THREADS + threadIdx.x;
  const int f = (v < V && lab[v] == v) ? 1 : 0;
  int total;
  const int ex = wlf_block_scan(f, &total, s_warp);
  if (f) rank[v] = block_sums[blockIdx.x] + ex;
}
__global__ void __launch_bounds__(256)
wl_dens_apply(int V, const int* __restrict__ lab, const int* __restrict__ rank, int* __restrict__ out) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v < V) out[v] = rank[lab[v]];
}

}  // namespace gk
