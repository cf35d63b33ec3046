// Shared declarations of the grakel_b200 CUDA library (sm_90a only).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>

#include <atomic>
#include <cstddef>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/grakel_b200.h"

namespace gk {

// ---------------------------------------------------------------- errors
extern thread_local std::string g_last_error;

inline int fail(int code, const std::string& msg) {
  g_last_error = msg;
  return code;
}

#define GK_CUDA(expr)                                                                      \
  do {                                                                                     \
    cudaError_t _e = (expr);                                                               \
    if (_e != cudaSuccess) {                                                               \
      return gk::fail(GK_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e) +   \
                                       " (" + __FILE__ + ":" + std::to_string(__LINE__) + ")"); \
    }                                                                                      \
  } while (0)

#define GK_TRY(expr)          \
  do {                        \
    int _r = (expr);          \
    if (_r != GK_OK) return _r; \
  } while (0)

// ---------------------------------------------------------------- buffers
// Bytes held by every DevBuf [0] / PinBuf [1] of the process; read by gk_selftest_live_bytes only.
extern std::atomic<int64_t> g_live_bytes[2];

// Grow-only buffer that owns its allocation: device memory (DevBuf) or pinned host staging (PinBuf: D2H of small
// scalars, H2D of CSR).  The engine is called repeatedly on same-sized workloads (bench loop, fit then transform), so
// capacity is kept between calls; the allocation is freed with the buffer.  Moves leave the source empty; a copy
// would free the allocation twice, so there is none.
template <bool Pinned>
struct Buf {
  void* p = nullptr;
  size_t cap = 0;
  Buf() = default;
  Buf(const Buf&) = delete;
  Buf& operator=(const Buf&) = delete;
  Buf(Buf&& o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
  Buf& operator=(Buf&& o) noexcept {
    if (this != &o) {
      free_block();
      p = o.p; cap = o.cap;
      o.p = nullptr; o.cap = 0;
    }
    return *this;
  }
  ~Buf() { free_block(); }
  int ensure(size_t bytes) {
    if (bytes <= cap) return GK_OK;
    free_block();
    const size_t want = Pinned ? bytes + 256 : bytes + (bytes >> 3) + 256;
    cudaError_t e = Pinned ? cudaMallocHost(&p, want) : cudaMalloc(&p, want);
    if (e != cudaSuccess) {
      p = nullptr;
      return fail(GK_ERR_CUDA, std::string(Pinned ? "cudaMallocHost(" : "cudaMalloc(") + std::to_string(want) +
                                   "): " + cudaGetErrorString(e));
    }
    cap = want;
    g_live_bytes[Pinned] += (int64_t)cap;
    return GK_OK;
  }
  template <class T>
  T* as() const { return reinterpret_cast<T*>(p); }

 private:
  void free_block() {
    if (p) {
      if (Pinned) cudaFreeHost(p);
      else cudaFree(p);
      g_live_bytes[Pinned] -= (int64_t)cap;
    }
    p = nullptr;
    cap = 0;
  }
};
using DevBuf = Buf<false>;
using PinBuf = Buf<true>;

constexpr unsigned long long EMPTY64 = ~0ULL;
constexpr int MAX_LEVELS = 64;

// Device-side scalars the pipeline reads back once per phase.
struct DevScalars {
  long long level_dims[MAX_LEVELS];      // distinct labels per WL level
  long long level_base[MAX_LEVELS + 1];  // first column id of each level
  unsigned int collision;                // WL: a hash collision was detected (-> retry with new seed)
  unsigned int ft_overflow;              // feature table probe overflow (cannot happen at load <= 0.5)
  unsigned long long n_entries;          // nnz of the feature block
  unsigned long long max_count;          // largest count
  unsigned long long max_diag;           // largest self similarity
  long long n_dense;                     // D_c
  unsigned long long sp_coo;             // wl_fused2: self-similarity units of frozen vertices (= sum of diag_frozen)
  unsigned int sp_dict_size;             // SP: number of distinct (lu,lv,d) keys
  unsigned int sp_nonint;                // SP: a non-integer / out-of-range distance was met
  unsigned int fattr_negative;           // SP-attr: the feature map has a negative entry
  unsigned int nh_order_dep;             // NeighborhoodHash: a count-sensitive result depended on the neighbour order
  unsigned int sp_dkey_size;             // SP real mode / SP-attr: number of distinct path-length bit patterns
  unsigned int pad0;
};

static_assert(sizeof(DevScalars) % 8 == 0, "cleared as 64-bit words");

constexpr int HIST_BUCKETS = 16;        // bucket b: 2^(b-1) < m <= 2^b ; last = saturated

struct ColStats {           // device-side, zeroed per gk_gram
  unsigned long long hist_cols[HIST_BUCKETS];
  unsigned long long hist_work[HIST_BUCKETS];
  unsigned long long hist_entries[HIST_BUCKETS];  // sum of m over the bucket's columns
  long long n_dense;        // D_c (head columns)
  long long n_tail_cols;
  long long n_tail_entries;
  long long tail_work;      // pair updates the tail kernel performs
  int T;                    // chosen threshold
  int pad;
};

// What the handle's feature block holds, i.e. which gk_gram route computes K from it.
enum FeatureKind : int {
  FK_NONE = 0,
  FK_WL = 1,      // WL / WL-OA / VertexHistogram / EdgeHistogram (graph, column) counts: the integer Gram
  FK_SP = 2,      // ShortestPath (lu, lv, d) counts: the integer Gram
  FK_SPATTR = 3,  // ShortestPathAttr dense fp64 feature matrix
  FK_GH = 4,      // GraphHopper per-vertex maps
  FK_NH = 5,      // NeighborhoodHash per-level expanded blocks
  FK_RW = 6,      // random walk edge values
  FK_PK = 7,      // Propagation counts in the SP layout: the integer Gram
  FK_PM = 8,      // PyramidMatch per-level expanded blocks (the NeighborhoodHash layout)
  FK_NSPD = 9,    // NeighborhoodSubgraphPairwiseDistance per-(radius, distance) count tables
  FK_SM = 10,     // SubgraphMatching per-graph bitset records
  FK_ODD = 11,    // OddSth per-bit-plane (graph, identity) count tables
  FK_ML = 12,     // MultiscaleLaplacian per-graph (S^-1, log det S) records
  FK_SVMT = 13,   // SvmTheta per-graph first-level phi
  FK_GS = 14,     // GraphletSampling (graph, class) counts: the integer Gram
};

}  // namespace gk

// The opaque handle of the C-ABI.
struct gk_handle {
  int dev = 0;
  int sm_count = 132;
  cudaStream_t stream = nullptr;
  cudaStream_t stream2 = nullptr;  // side stream: independent kernels of one phase run concurrently
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  cudaEvent_t ev_stage[4] = {};  // D2H staging ring of host_deliver.h
  cudaEvent_t ev[16] = {};
  cudaEvent_t tev[8] = {};  // internal stage timers

  // ---- packed graphs
  int64_t N = 0, V = 0, E = 0;
  int32_t n_labels0 = 0;
  bool has_weights = false, unit_weights = true;
  int32_t attr_dim = 0;
  int32_t max_degree = 0, max_graph_size = 0;
  gk::DevBuf graph_ptr, row_ptr, col_idx, labels0, weights, attrs, vgraph;
  std::vector<int> graph_ptr_host;
  std::vector<int> graph_eptr_host;  // first edge of each graph (row_ptr[graph_ptr[g]])
  bool has_labels = false;  // the current block was packed with vertex labels (labels0 may hold an older block's)
  gk::DevBuf sp_lists;      // graph lists of the shortest-path launches (kept apart from large_list: gk_wl_features reads that)
  gk::DevBuf large_list;  // vertices with degree > group width
  int64_t n_large = 0;
  int group_width = 32;

  // ---- WL scratch
  int n_levels = 0;
  gk::DevBuf labels_all;  // [(h+1) * V] int32
  gk::DevBuf sig_nbr;     // [E] sorted neighbour labels of the current level
  gk::DevBuf slot_of;     // [V] hash slot, then representative vertex
  gk::DevBuf ht_keys, ht_rep;
  size_t ht_cap = 0;
  gk::DevBuf flags, block_sums;
  gk::DevBuf wlf_buf;  // fused WL kernel: [tile_vbeg (T+1) | cta_tile (G+1) | barrier]
  // fused WL kernel: the tile partition of the packed block (device copy in wlf_buf) is kept between calls
  bool wl_tiles_valid = false;
  bool wl_tiles_fused = false;
  int wl_n_tiles = 0;
  long long wl_tiles_key = -1;  // GRAKEL_B200_WL_TILES_PER_CTA the partition was built with
  gk::DevBuf wl_payload;  // fused WL kernel: [2][ht_cap] 32-byte slot payloads (the installing vertex's signature)
  gk::DevBuf wl_single;  // fused WL kernel: one byte per vertex (frozen flag)
  gk::DevBuf diag_frozen;  // fused WL kernel: frozen vertices' share of the self similarities (u64 per graph)
  bool wl_sparse_ids = false;  // labels of levels >= 1 are representative vertex ids (wl_fused2), not dense ranks
  gk::DevBuf scalars;  // gk::DevScalars
  gk::PinBuf h_scalars;

  // ---- feature block (hash table of (graph, column) -> count)
  gk::DevBuf ft_keys, ft_cnt;
  size_t ft_cap = 0;
  int64_t n_columns = 0;
  // the complete feature block the handle holds, FK_NONE for none: a feature pass clears it when it starts and sets it
  // as its last step (features_begin / features_publish in api.cu), so a pass that fails in between leaves no block
  gk::FeatureKind feature_kind = gk::FK_NONE;
  bool pro_ready = false;  // the pass that published the block also ran its square Gram prologue (gk_wl_features,
                           // the asynchronous WL pass): self similarities finished, column histogram on the host --
                           // gk_gram then needs no host synchronisation before its launches
  // the Gram prologue's results that gk_gram would otherwise read back after a synchronisation
  gk::ColStats pro_hist;
  long long pro_max_count = 0, pro_max_diag = 0, pro_n_entries = 0;

  gk::DevBuf oa_keys, oa_cnt, oa_colcnt;  // WL-OA: unary-expanded block, swapped with ft_keys / ft_cnt / colcnt
  // ---- columns / panel / diag
  gk::DevBuf colcnt, colmin, colmax, colslot, col_flags3, col_block_sums, colstats;
  int64_t col_cap = 0;  // allocated length of the per-column arrays
  gk::DevBuf part_max, part_new;  // per-CTA partials of the feature kernels
  int64_t n_part = 0;
  gk::DevBuf tail_desc, tail_ent, tail_cur;
  gk::PinBuf h_colstats;
  gk::DevBuf tb_cnt, tb_ent, tb_ovf;  // tail fused into the GEMM epilogue: per-block update lists + overflow (features.cuh tail_bucket)
  gk::DevBuf gram_dyn;   // gk::GramDyn: device-side decisions of the asynchronous pass (gk_wl_gram)
  gk::PinBuf h_dyn;
  gk::DevBuf diag_u64, diag_f64;
  gk::DevBuf row_map, diag_rows;  // gk_set_row_map: packed graph -> row of K (0 rows = identity)
  int64_t n_rows = 0;
  gk::DevBuf panel;
  int64_t Dc = 0, Dc_pad = 0;

  // ---- SP scratch
  gk::DevBuf sp_dist;      // global-memory distance matrices for graphs too large for smem
  gk::DevBuf sp_dict_keys; // (lu,lv,d) -> column dictionary
  gk::DevBuf sp_dict_ids;
  gk::DevBuf sp_dkeys;     // real-valued weights: dictionary of distance bit patterns
  size_t sp_dict_cap = 0;
  gk::DevBuf sp_graph_off; // per-graph offset into sp_dist (for gk_sp_distances)
  std::vector<long long> sp_goff;  // its host copy
  int sp_flags = 0;
  int sp_dist_esz = 0;     // gk_spattr_features: element size of the matrices it left in sp_dist (2 = u16, 8 = fp64)

  // ---- SP-attr dense fp64 feature matrix
  gk::DevBuf fattr;
  int64_t fattr_dim = 0;
  bool fattr_signed = false;  // some feature is negative: entries of K may cancel (gram_spattr takes the fp64 Gram)

  // ---- GraphHopper (FK_GH): per-vertex maps M [V][delta (delta + 1) / 2] fp64
  gk::DevBuf gh_M, gh_ws, gh_woff, gh_gdiam, gh_groups, gh_pairs;
  int gh_delta = 0;
  int gh_node_kernel = 0;  // GK_GH_LINEAR / GK_GH_GAUSSIAN / GK_GH_BRIDGE
  double gh_mu = 1.0;

  // ---- NeighborhoodHash (FK_NH)
  gk::DevBuf nh_codes, nh_valid;  // [(R + 1) V] u64 codes / u8 not-None flags: the initial labels, then levels 0 .. R-1
  gk::DevBuf nh_blk;              // unary-expanded (graph, column) block of every level, nh_level_bytes apart
  gk::DevBuf nh_lut, nh_tab, nh_ws, nh_cur, nh_C;
  size_t nh_level_bytes = 0;
  int64_t nh_level_cap = 0;       // entries (and columns) one level's expanded block can hold
  int nh_R = 0;
  std::vector<long long> nh_dims, nh_cols, nh_entries;  // per level: distinct codes, columns and entries of its block

  // ---- PyramidMatch (FK_PM): the levels live in the NeighborhoodHash buffers above (nh_codes / nh_valid hold the
  // current level's keys, nh_blk the expanded blocks, pm_S * pm_L of them); the embeddings [S][V][d] fp64 and the
  // column counts [S][N] stay for gk_pm_cells and the self similarities
  gk::DevBuf pm_U, pm_ncols, pm_skip;  // pm_skip: [V] u8, vertices without entries (when has_skip)
  int pm_S = 0, pm_L = 0, pm_d = 0, pm_flags = 0;
  bool pm_has_skip = false;

  // ---- HadamardCode (an FK_WL or FK_SP block): the two level buffers of V x W u64 vectors, the hash multipliers, the
  // skip flags and the shape of the last gk_hc_features call (gk_hc_vectors recomputes its levels from them)
  gk::DevBuf hc_S, hc_z, hc_skip;
  int hc_W = 0, hc_levels = 0;
  bool hc_has_skip = false;
  bool hc_degenerate_once = false;  // gk_selftest_hc_collision: the next pass starts with all z_c = 0
  // gk_selftest_wl_collision: the next wl_degen_attempts WL relabel attempts hash (own label, degree) only at the levels
  // >= wl_degen_from
  int wl_degen_attempts = 0, wl_degen_from = 1;

  // ---- NeighborhoodSubgraphPairwiseDistance (FK_NSPD): BFS level matrices [sum n_g^2] u8 and their queue, hashes
  // [(r + 1) V] u32, the host tables (aux), the hashing slots, the pairs of every distance, the per-level (graph,
  // column) count tables and the fp64 count matrix of one level
  gk::DevBuf nspd_lvl, nspd_q, nspd_H, nspd_aux, nspd_ws, nspd_pairs, nspd_blk, nspd_tab, nspd_keys, nspd_C;
  int nspd_r = 0, nspd_d = 0;
  // per level (delta-major): its table's byte offset in nspd_blk, slots, pairs and columns; per graph, the mask of the
  // distances it has pairs at
  std::vector<long long> nspd_off, nspd_cap, nspd_M, nspd_cols;
  std::vector<unsigned long long> nspd_mask;

  // ---- WL over a base kernel whose levels cannot share one feature block (gk_wl_level_sum): the running fp64 sum of
  // the levels' K and the K of the current level; shape and square-ness of the sum, levels added so far.  No re-pack or
  // feature pass touches them, so the sum survives the per-level gk_pack_csr / gk_nspd_features calls.
  gk::DevBuf wl_sum, wl_lvl;
  int64_t wl_sum_rows = 0, wl_sum_cols = 0, wl_sum_row0 = 0;
  int32_t wl_sum_levels = 0;
  bool wl_sum_square = false;
  // CoreFramework reuses the sum (gk_core_sum_begin / gk_core_level_add): the sum is a core fold, the last core level
  // added (levels go strictly downwards), the level's row and column maps
  bool core_sum = false;
  int32_t core_level = 0;
  gk::DevBuf core_map;

  // ---- random walk (FK_RW): edge values of the packed CSR, its transpose, eigen-data, coefficients
  gk::DevBuf rw_val, rw_trp, rw_tci, rw_tval, rw_q, rw_w, rw_coef, rw_ws, rw_iters, rw_cap;
  int rw_route = 0, rw_fn = 0, rw_ncoef = 0;
  double rw_lamda = 0.0;
  bool rw_labeled = false;
  int64_t rw_iter_rows = 0, rw_iter_cols = 0;  // shape of the iteration counts of the last gk_gram

  // ---- SubgraphMatching (FK_SM): per-graph records and their offsets, edge label ids, weight tables, lambdas, the
  // extension-set stacks, [pair counter u64 | error bits u32 | largest neighbour count u32]
  gk::DevBuf sm_rec, sm_off, sm_el, sm_vtab, sm_etab, sm_lam, sm_stack, sm_ctl;
  int sm_k = 0, sm_kk = 1, sm_kv = 0, sm_ke = 0, sm_n_vl = 0, sm_n_el = 0;
  int sm_max_und = 0;  // largest number of distinct out- or in-neighbours of a packed vertex
  gk::DevBuf sm_wl_cls;  // gk_sm_wl_features: sm_n_lv WL class ids per packed vertex (0 levels: plain SubgraphMatching)
  int sm_n_lv = 0;
  bool sm_hc = false;    // gk_sm_hc_features: sm_wl_cls holds HadamardCode classes (levels need not refine)
  bool sm_exact = true;

  // ---- OddSth (FK_ODD): graph offsets and label ranks, node records [S] (hash | label | graph | first child | child
  // count | slot | identity), children [T], the interning table, per-identity arrays (representative | C | plane
  // column), the (graph, identity) counts, the bit-plane tables, counters, self similarities
  gk::DevBuf odd_aux, odd_nodes, odd_ch, odd_tab, odd_feat, odd_phi, odd_blk, odd_ctl, odd_diag;
  int odd_degen = 0;  // gk_selftest_odd_collision: degenerate identity passes still to come
  // node slots, child slots, identities; per bit plane of C, its table's byte offset in odd_blk, slots, entries and
  // columns
  long long odd_S = 0, odd_T = 0, odd_F = 0, odd_maxC = 0;
  std::vector<long long> odd_off, odd_cap, odd_M, odd_cols;

  // ---- MultiscaleLaplacian (FK_ML): dense per-graph adjacency and its offsets, radius-l ball masks [L][V][2], the
  // features of the current level and their successor, vertex records [V][P' P' + 1], the sample records of the current
  // level, sample ids / Q scratch, error bits; after gk_ml_finish ml_rec holds the Gram's records (fitted ones first)
  gk::DevBuf ml_adj, ml_adj_off, ml_ball, ml_U, ml_U2, ml_vrec, ml_samp, ml_rec, ml_aux, ml_ctl;
  int ml_L = 0, ml_w = 0, ml_mcap[65] = {};
  double ml_gamma = 0.0, ml_heta = 0.0;
  int64_t ml_nrec = 0;

  // ---- SvmTheta (FK_SVMT): vertex offsets, out-edge bitmask rows [V][4], smallest eigenvalues, alphas [V], iteration
  // counts, schedule / draw / sum offsets, drawn indexes, sample sums, phi [N][L], error bits; svmt_rec holds the Gram's
  // first-level phi (fitted graphs first)
  gk::DevBuf svmt_vptr, svmt_adj, svmt_m, svmt_alpha, svmt_iters, svmt_cnt, svmt_off, svmt_idx, svmt_sums, svmt_phi,
      svmt_rec, svmt_ctl;
  std::vector<int> svmt_sizes;  // vertices of the graphs of the last gk_svmt_solve
  int64_t svmt_nrec = 0;

  // ---- GraphletSampling (FK_GS): the canonical class table of the code space (built once, for sizes up to gs_canon_k),
  // the first graph of every class among the fitted / the new graphs, class -> column, the (graph, column) table with
  // its sample counts and class codes, graphs per column, self similarities, [error bits | pad | columns u64 | max, entries]
  gk::DevBuf gs_canon, gs_first, gs_colid, gs_blk, gs_colcnt, gs_diag, gs_ctl, gs_samp;
  int gs_canon_k = 0;
  size_t gs_cap = 0;
  int64_t gs_cols = 0;

  // ---- Propagation (FK_PK): P double-buffered [2][V][D], every level's bins [t_max][V][K], the private
  // flags of every level [t_max][V], per-edge T values, draws, column scratch, counters [near u64 | nan u32 | pad]
  gk::DevBuf pk_P, pk_bins, pk_priv, pk_tval, pk_u, pk_b, pk_tab, pk_cnt;
  int pk_levels = 0, pk_K = 0;

  // ---- GEMM
  gk::DevBuf tiles;  // int2 list: rebuilt and uploaded only when its key changes
  long long tiles_key[8] = {-1, -1, -1, -1, -1, -1, -1, -1};
  long long tiles_n = 0;
  long long head_row_bytes = 0;  // panel row width (bytes) of the last pass whose threshold came from the cost model
                                 // (not GK_DENSE_ALL / FORCE_T)
  long long last_max_count = 0;  // largest count of the last Gram on this handle: an asynchronous pass fills a u8 panel
                                 // unless it was 256 (a count of 256 repeats through the synchronous route once)
  gk::PinBuf h_tiles;
  gk::PinBuf h_bands;  // band table of the u16 result transport (its own buffer: h_tiles may still feed an async copy)
  gk::DevBuf K;      // device-resident result of the last gk_gram
  int64_t K_rows = 0, K_cols = 0, K_ld = 0;  // K_ld: row pitch in elements (>= K_cols)
  int K_dtype = GK_F32;
  gk::DevBuf K_stage;  // fp64 staging when K is kept as f32 but fetched as f64

  gk::PinBuf h_stage;  // pinned staging ring of the result delivery
  gk::PinBuf h_diag;   // self similarities on the host (normalisation during the widening)
  int64_t launches = 0;
  void* comm = nullptr;  // gk::Comm (comm.h) after gk_comm_init

  // Runs before any member is destroyed: the communicator's collective teardown (every peer unmaps this handle's
  // exported blocks) completes before the buffers free themselves.  The null checks keep a partly built handle from
  // leaving an error behind for the next cudaGetLastError on this thread.
  ~gk_handle() {
    cudaSetDevice(dev);
    if (stream) cudaStreamSynchronize(stream);
    gk_comm_destroy(this);
    for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e);
    for (cudaEvent_t e : tev) if (e) cudaEventDestroy(e);
    for (cudaEvent_t e : ev_stage) if (e) cudaEventDestroy(e);
    if (ev_fork) cudaEventDestroy(ev_fork);
    if (ev_join) cudaEventDestroy(ev_join);
    if (stream) cudaStreamDestroy(stream);
    if (stream2) cudaStreamDestroy(stream2);
  }
};
