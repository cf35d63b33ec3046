/* grakel_b200 -- C-ABI of the H100-native graph-kernel Gram engine.
 *
 * This header is the drop-in boundary for the hot path of ysig/GraKeL
 * (reference v0.1.11):  N x N Gram matrices of the Weisfeiler-Lehman subtree
 * kernel and the Shortest-Path kernels.  The reference has no FFI on this path
 * (it is pure Python + numpy/scipy); its only native precedent is the Cython
 * `cdef extern` block grakel/kernels/_c_functions/header.pxd:1-4 over
 * include/functions.hpp:4-5 (raw pointers + sizes, results by out-pointer).
 * The entry points below follow that convention: extern "C", plain pointers and
 * sizes, caller-owned host buffers, library-owned device memory behind an
 * opaque handle, int status return (0 = ok, <0 = error; text via gk_last_error).
 *
 * What each entry point replaces in the reference:
 *
 *   gk_pack_csr          Graph.__init__/build_graph/_import_*  (graph.py:147-230,
 *                        912-1053) + get_edge_dictionary/get_labels
 *                        (graph.py:1182-1204, 689-772) -- after the Python layer
 *                        has normalised the input into one CSR block.
 *   gk_wl_features       WeisfeilerLehman.parse_input relabel loop
 *                        (weisfeiler_lehman.py:199-258) + VertexHistogram.parse_input
 *                        (vertex_histogram.py:57-154) for every level.
 *   gk_sp_features       Graph.build_shortest_path_matrix / floyd_warshall / dijkstra
 *                        (graph.py:588-687, 1712-1794) + ShortestPath.parse_input
 *                        pair histogram (shortest_path.py:468-490).
 *   gk_wl_sp_features    the WL level loop with ShortestPath as base kernel
 *                        (weisfeiler_lehman.py:260-270, "WL-SP" of doc/benchmarks).
 *   gk_wl_oa_features    WeisfeilerLehmanOptimalAssignment.parse_input + the O(N^2) Python loop of
 *                        histogram intersections (weisfeiler_lehman_optimal_assignment.py:78-229,
 *                        257-266, 433-437).
 *   gk_spattr_features   ShortestPathAttr.parse_input + the bilinear pair kernel
 *                        (shortest_path.py:77-164) as an explicit feature map.
 *   gk_gram              VertexHistogram._calculate_kernel_matrix
 *                        (vertex_histogram.py:156-184), np.sum over levels
 *                        (weisfeiler_lehman.py:270), np.dot(phi, phi.T)
 *                        (shortest_path.py:404 / :312), the diagonals
 *                        (vertex_histogram.py:186-219, shortest_path.py:320-368) and
 *                        the normalisation (weisfeiler_lehman.py:324-327, 494-498;
 *                        shortest_path.py:314-316, 407-408).
 *   gk_wl_fit_transform, gk_sp_fit_transform
 *                        one-call forms of the above with HOST buffers in and out:
 *                        WeisfeilerLehman.fit_transform (weisfeiler_lehman.py:292-328),
 *                        ShortestPath.fit_transform (shortest_path.py:370-410).
 *
 * Fit + transform.  The reference keeps per-level dictionaries at fit time and
 * re-applies them to new graphs (weisfeiler_lehman.py:330-500).  Here the same
 * result is obtained by packing the fitted graphs X followed by the new graphs Y
 * into one block and relabelling them jointly: a Y feature is "seen" iff its
 * column also occurs in an X graph, unseen columns contribute nothing to
 * K[y, x] and are counted in Y's self-similarity, exactly as
 * vertex_histogram.py:179 / :211-217 and shortest_path.py:312 / :365 do.
 * `n_fit` below is the number of leading graphs that form X.
 */
#ifndef GRAKEL_B200_H
#define GRAKEL_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct gk_handle gk_handle;

/* output element type of K */
#define GK_F32 0
#define GK_F64 1

/* gk_gram flags */
#define GK_NORMALIZE 1   /* K_ij / sqrt(d_i d_j) in fp64 (weisfeiler_lehman.py:326) */
#define GK_NAN_TO_NUM 2  /* WL only: np.nan_to_num on the normalised matrix          */
#define GK_GRAM_SIMT 4   /* use the exact int64 CUDA-core Gram (verification / wide counts) */
#define GK_OUT_DEVICE 8  /* K_out is a DEVICE pointer (e.g. a torch tensor)          */
#define GK_FULL_TILES 16 /* square case: compute every tile, no mirroring            */
#define GK_DENSE_ALL 32  /* contract every shared column on the tensor cores (no sparse tail) */

/* gk_sp_features flags */
#define GK_SP_WITH_LABELS 1
#define GK_SP_KEEP_DIST 2    /* keep fp64 APSP matrices for gk_sp_distances (tests) */
#define GK_SP_DIJKSTRA_ORDER 4 /* real-valued weights: path sums associate as in dijkstra (graph.py:1712-1764), not as in
                                floyd_warshall (:1767-1794); integer-valued distances are the same either way */

/* error codes */
#define GK_OK 0
#define GK_ERR_CUDA -1
#define GK_ERR_ARG -2
#define GK_ERR_STATE -3
#define GK_ERR_RANGE -4   /* a count or Gram value leaves the exactly representable range */
#define GK_ERR_UNSUPPORTED -5

/* Per-call statistics (all optional; pass NULL).  Times are CUDA-event
 * milliseconds on the handle's stream. */
typedef struct gk_stats {
  int64_t n_graphs, n_vertices, n_edges;
  int64_t n_levels;          /* WL: h+1 */
  int64_t level_dims[64];    /* WL: distinct labels per level (= D_i of the reference) */
  int64_t n_columns;         /* total feature columns D */
  int64_t n_entries;         /* nnz of the feature block */
  int64_t n_dense_columns;   /* D_c: "head" columns contracted by the tensor-core GEMM */
  int64_t n_tail_columns;    /* low-frequency columns contracted by exact atomic pair updates */
  int64_t tail_updates;      /* number of those pair updates */
  int64_t threshold;         /* T: columns in more than T graphs are head columns */
  int64_t max_count;         /* largest single feature count */
  int64_t max_diag;          /* largest self-similarity */
  int64_t hash_retries;      /* WL: relabel passes repeated after a detected hash collision */
  int64_t gram_path;         /* 1 = wgmma tensor-core GEMM over the integer panel (u8 or bf16: gemm_elem_bytes), 2 = exact int64 CUDA-core Gram, 3 = no contracted columns,
                                ShortestPathAttr: 4 = 3xTF32 wgmma GEMM (non-negative features), 5 = fp64 CUDA-core Gram,
                                GraphHopper node-pair kernels: 6 = fused fp64 CUDA-core node-pair Gram,
                                NeighborhoodHash: 7 = one exact integer Gram per level + the fp64 combine,
                                random walk: 8 = conjugate gradients, 9 = spectral pair sum, 10 = power series,
                                PyramidMatch: 11 = one exact integer Gram per level + the fp64 combine,
                                NeighborhoodSubgraphPairwiseDistance: 12 = one exact integer Gram per level + the fp64 fold,
                                SubgraphMatching: 13 = per-pair clique counts + the lambda fold,
                                OddSth: 14 = one exact integer Gram per bit of C + the fp64 sum of 2^b G_b,
                                MultiscaleLaplacian: 15 = per-pair FLG values, SvmTheta: 16 = fp64 product of first-level phi,
                                GraphletSampling: 17 = the exact integer Gram of the (graph, class) counts */
  int64_t gemm_tiles;        /* output tiles computed */
  int64_t gemm_launches;     /* kernels launched by the last gk_gram */
  int64_t kernel_launches;   /* kernels launched by the last features call */
  float ms_h2d, ms_features, ms_panel, ms_gemm, ms_tail, ms_d2h, ms_total;
  int64_t gemm_elem_bytes;   /* element bytes of the integer head panel the tensor-core GEMM (gram_path 1) read:
                                1 = u8 (u8 x u8 -> s32 wgmma, every count <= 255), 2 = bf16 (a count of 256, or
                                GRAKEL_B200_U8=0), 0 = no integer tensor-core GEMM ran */
  /* NeighborhoodHash: gk_nh_features' hash levels and per-level columns + unary expansion; gk_gram's combine and
     the integer Gram of every level */
  float ms_hash, ms_columns, ms_combine;
  float ms_level_gram[64];
  int64_t nh_order_dependent; /* NeighborhoodHash, count sensitive: some vertex had two different neighbour codes with
                                 equal low `bits` bits, so its code depended on the order of its neighbours */
  /* random walk: device time of gk_gram's pair kernels (self similarities included), and the Taylor pairs that
     stopped at the term cap before converging */
  float ms_rw;
  int64_t rw_cap_hits;
  /* Propagation: device time of the P <- T P steps (inside ms_hash, which covers propagation + hashing), and the
     hashes (or float32 / integer stores of P) within 2^-30 of their magnitude of a bin edge, where a different
     summation order could move a vertex to the neighbouring bin */
  float ms_propagate;
  int64_t pk_near_edge;
} gk_stats;

int gk_version(void);
const char* gk_last_error(void);

int gk_create(int device_ordinal, gk_handle** out);
int gk_destroy(gk_handle* h);
int gk_sync(gk_handle* h);

/* Upload one packed CSR block (host pointers).
 *   graph_ptr[n_graphs+1]  vertex offsets, graph g owns vertices [graph_ptr[g], graph_ptr[g+1])
 *   row_ptr[V+1]           out-edge offsets per vertex (V = graph_ptr[n_graphs])
 *   col_idx[E]             GLOBAL vertex id of each out-neighbour (same graph)
 *   labels[V]              dense non-negative id of the vertex label (level 0), or NULL
 *   weights[E]             edge weights (fp64) or NULL for unit weights
 *   attrs[V*attr_dim]      fp64 node attributes or NULL                                  */
int gk_pack_csr(gk_handle* h, int64_t n_graphs, const int32_t* graph_ptr, const int32_t* row_ptr,
                const int32_t* col_idx, const int32_t* labels, const double* weights,
                const double* attrs, int32_t attr_dim);

/* Build the sparse feature block of the packed graphs on the device. */
int gk_wl_features(gk_handle* h, int32_t n_iter, gk_stats* stats);
int gk_sp_features(gk_handle* h, int32_t flags, gk_stats* stats);
int gk_spattr_features(gk_handle* h, int32_t flags /* GK_SP_DIJKSTRA_ORDER or 0 */, gk_stats* stats);
/* WeisfeilerLehman(base_graph_kernel=ShortestPath), weisfeiler_lehman.py:260-270 over
 * shortest_path.py:370-410: n_iter WL rounds, then the labelled shortest-path histogram of every
 * level in one feature block (level-unique label ids => disjoint columns), so that one gk_gram
 * returns the sum of the per-level matrices. */
int gk_wl_sp_features(gk_handle* h, int32_t n_iter, int32_t flags, gk_stats* stats);

/* WeisfeilerLehmanOptimalAssignment (weisfeiler_lehman_optimal_assignment.py:78-279): the WL feature
 * block of all levels in unary ("thermometer") form -- column c with count k becomes k columns holding 1
 * -- so that gk_gram's dot products are the histogram intersections sum_c min(Hs[i,c], Hs[j,c]) of
 * :257-266 / :433-437, the self similarities the row sums of :459-461, exactly (integers). */
int gk_wl_oa_features(gk_handle* h, int32_t n_iter, gk_stats* stats);

/* GraphHopper (graph_hopper.py:19-449): per-vertex maps M_v (delta x delta, delta = largest diameter + 1 over the
 * packed block) from the shortest-path DAG of every root, then the node kernel:
 *   GK_GH_LINEAR    <x, x'>: explicit feature map Phi(G) = sum_v vec(M_v) (x) x_v; gk_gram takes the ShortestPathAttr
 *                   Gram (gram_path 4 = 3xTF32 for non-negative attributes, 5 = fp64 for attributes of mixed sign)
 *   GK_GH_GAUSSIAN  exp(-mu ||x - x'||^2)
 *   GK_GH_BRIDGE    max(0, (4 - ||x - x'||) / 4)
 *                   both: fused fp64 node-pair Gram (gram_path 6), exactly symmetric and deterministic
 * Unit edge weights only (GK_ERR_UNSUPPORTED otherwise); node attributes are required; flags must be 0.
 * stats: level_dims[0] = delta, n_columns = feature dimension (linear) or delta (delta + 1) / 2 (node-pair kernels).
 * gk_gram: fp64 host output, GK_NORMALIZE, n_fit and row ranges; GK_DIST is GK_ERR_UNSUPPORTED. */
#define GK_GH_LINEAR 0
#define GK_GH_GAUSSIAN 1
#define GK_GH_BRIDGE 2
int gk_gh_features(gk_handle* h, int32_t node_kernel, double mu, int32_t flags, gk_stats* stats);
/* graph g's maps after gk_gh_features: out[n * delta * delta], M[v][a][b] at (v * delta + a) * delta + b */
int gk_gh_node_maps(gk_handle* h, int64_t g, double* out);

/* NeighborhoodHash (neighborhood_hash.py:14-570): R levels of neighbourhood hashing of u64 codes over the
 * out-neighbours of the packed block, level 0 hashing the initial codes.  The packed label ids index
 * code_of_label[n_labels] (the initial code of every label id) and label_valid[n_labels] (0 = None: a label unseen at
 * fit; NULL = all valid).  bits in [1, 64] (masked rotations as in the reference's ROT).  A vertex whose code or any
 * neighbour's code is None is None.  Count sensitive: runs of equal codes after a stable sort of each row by the low
 * `bits` bits, as the reference's radix_sort_rot -- so each row must list its neighbours in the order of the
 * reference's edge dictionary.  Every level's non-None codes become one unary-expanded count block of its own.
 * stats: level_dims[r] = distinct codes of level r, n_columns = expanded columns of all levels, ms_hash / ms_columns.
 * gk_gram then returns K_ij = sum(t_r) / R (CPython's float sum) with t_r = c_r / (n_i + n_j - c_r), c_r the multiset
 * intersection of the two graphs' non-None level-r codes and n the graphs' vertex counts (gram_path 7): fp64 only,
 * host or GK_OUT_DEVICE output, n_fit and row ranges; xdiag / ydiag are 1; GK_NORMALIZE has no effect; GK_DIST and
 * row maps are GK_ERR_UNSUPPORTED.  flags must be 0. */
#define GK_NH_SIMPLE 0
#define GK_NH_COUNT_SENSITIVE 1
int gk_nh_features(gk_handle* h, int32_t R, int32_t nh_type, int32_t bits, const uint64_t* code_of_label,
                   const uint8_t* label_valid, int64_t n_labels, int32_t flags, gk_stats* stats);
/* codes of level `level` (0 .. R-1) of every packed vertex after gk_nh_features: out[V] u64, valid[V] (may be NULL) */
int gk_nh_labels(gk_handle* h, int32_t level, uint64_t* out, uint8_t* valid);

/* NeighborhoodSubgraphPairwiseDistance (neighborhood_subgraph_pairwise_distance.py).  The packed block lists every
 * graph's vertices in the reference's sorted-symbol order with ascending CSR columns (directed edges kept); labels
 * are vertex label ids.  sym_hash[V] = hash() of every vertex symbol, edge_label[E] = edge label id of every CSR
 * edge.  Tokens: tok_rank[(d + 1) * n_labels] is the rank of str(delta) + "," + str(label) in Python's string order;
 * rank_off[n_ranks + 1] / rank_bytes / rank_cp give every rank's UTF-8 bytes and code points, el_off[n_elabels + 1] /
 * el_bytes / el_cp those of str(edge label).  Builds the hashes H[rho][v] (BFS levels, CPython set order of the
 * sub-edge sets, APHash over the first code-point-count bytes of the encoding) and one (graph, column) count table
 * per level (delta, rho), levels numbered delta * (r + 1) + rho.  delta_mask[N] (may be NULL) receives the distances
 * every graph has pairs at.  (r + 1)(d + 1) > 64 is GK_ERR_UNSUPPORTED.  stats: level_dims = columns per level,
 * ms_hash (BFS levels + hashes) / ms_columns.  gk_gram (gram_path 12) then returns the reference's fp64 sum
 * of cosine-normalised level Grams over the fitted levels (square) or the levels both sides have (transform);
 * GK_NORMALIZE divides by the number of fitted levels, or sqrt(levels of Y x levels of X); xdiag / ydiag are those
 * level counts.  fp64 only, host or GK_OUT_DEVICE output, n_fit and row ranges; GK_DIST and row maps are
 * GK_ERR_UNSUPPORTED.  flags must be 0. */
int gk_nspd_features(gk_handle* h, int32_t r, int32_t d, const int64_t* sym_hash, const int32_t* edge_label,
                     const int32_t* tok_rank, int64_t n_labels, const int64_t* rank_off, const uint8_t* rank_bytes,
                     const int32_t* rank_cp, int32_t n_ranks, const int64_t* el_off, const uint8_t* el_bytes,
                     const int32_t* el_cp, int32_t n_elabels, uint64_t* delta_mask, int32_t flags, gk_stats* stats);
/* H[radius][v] of every packed vertex after gk_nspd_features: out[V] */
int gk_nspd_hashes(gk_handle* h, int32_t radius, uint32_t* out);
/* host only: the iteration order of CPython's set after inserting the n distinct pairs (h0[k], h1[k]) (element
 * hashes) in order k = 0 .. n-1 */
int gk_selftest_nspd_set_order(int64_t n, const int64_t* h0, const int64_t* h1, int64_t* order);

/* WeisfeilerLehman over NeighborhoodSubgraphPairwiseDistance: every WL level's K is a sum of cosine-normalised level
 * Grams, so the levels are added as matrices.  For level = 0, 1, ... in order: pack the level's labels, run
 * gk_nspd_features, then gk_wl_level_sum folds the level's K (gram_path 12, un-normalised; n_fit and the row range as in
 * gk_gram) into a device-resident fp64 sum, sum = sum + K_level, which rounds as numpy's np.sum(axis=0).  No re-pack or
 * feature pass touches the sum.  gk_wl_level_sum_fetch then applies GK_NORMALIZE (and GK_NAN_TO_NUM) with the self
 * similarities xdiag (the columns) and ydiag (a transform's rows; a square sum takes its rows' from xdiag), or with the
 * sum's own diagonal when xdiag is NULL (full square sum only), and copies K (rows x cols, row-major) to the host
 * array K_out; kdiag (may be NULL) receives the sum's diagonal before normalisation (full square sum only). */
int gk_wl_level_sum(gk_handle* h, int32_t level, int64_t n_fit, int64_t row_begin, int64_t row_end, gk_stats* stats);
int gk_wl_level_sum_fetch(gk_handle* h, int32_t flags, const double* xdiag, const double* ydiag, double* K_out,
                          double* kdiag);

/* CoreFramework over a base kernel whose core levels cannot share one feature block: the reference's
 * K[idx_j, idx] += K_i[j, :] for every core level i from the largest down (core_framework.py:177-223), on the device.
 * gk_core_sum_begin sizes the sum of gk_wl_level_sum (n_rows x n_cols fp64, row-major) and sets it to zero; `square`
 * marks a fit_transform sum, whose own diagonal gk_wl_level_sum_fetch may then read.  For each level: pack the level's
 * graphs, run the base kernel's feature pass, then gk_core_level_add computes the level's un-normalised K (the packed
 * feature kind's gram path, n_fit as in gk_gram, all rows; xdiag / ydiag as in gk_gram, may be NULL) into a
 * handle-owned buffer and adds it into the sum, sum[rows[j], cols[c]] += K_level[j, c], rows[n_level_rows] and
 * cols[n_fit] being distinct indices of the sum.  Levels must come in strictly descending order.  Every argument is
 * checked before the first launch.  No re-pack or feature pass touches the sum; gk_wl_level_sum_fetch then normalises
 * and copies it out once. */
int gk_core_sum_begin(gk_handle* h, int64_t n_rows, int64_t n_cols, int32_t square);
int gk_core_level_add(gk_handle* h, int32_t level, int64_t n_fit, int64_t n_level_rows, const int32_t* rows,
                      const int32_t* cols, double* xdiag, double* ydiag, gk_stats* stats);

/* RandomWalk / RandomWalkLabeled (random_walk.py:28-541), one graph pair per CTA in fp64.  The packed CSR gives the
 * structure (gk_pack_csr without weights; with labels for GK_RW_LABELED), `values[E]` the adjacency entries of its
 * edges (any sign, self-loops included), `t_row_ptr[V+1]` / `t_col_idx[E]` / `t_values[E]` the same block transposed
 * (in-edges, GLOBAL vertex ids).  Routes:
 *   GK_RW_CG        fn GK_RW_INV: scipy's cg(I - lamda M, 1, rtol=1e-6, maxiter=20) per pair, K = sum(x) (gram_path 8);
 *                   M p = Ax P Ay with P the Fortran-order reshape of p, masked as the reference's label-pair sum
 *   GK_RW_SPECTRAL  sum_ab (q_a q'_b)^2 f(w_a w'_b), q[V] / w[V] the per-graph eigen-data from the host (gram_path 9);
 *                   fn GK_RW_FINITE (coef[n_coef] = mu_0..mu_p, the reference's D *= Dij; S += mu_k D), GK_RW_EXP
 *                   exp(lamda z), GK_RW_INV 1 / (1 - lamda z); unlabelled only
 *   GK_RW_SERIES    sum_k c_k 1^T M^k 1 with M = D kron(Ax, Ay) D (gram_path 10): fn GK_RW_FINITE (c_k = coef[k]) or
 *                   GK_RW_EXP (c_k = lamda^k / k!, non-negative entries; pairs that reach the term cap are counted in
 *                   stats->rw_cap_hits)
 * gk_gram: fp64 only, host or GK_OUT_DEVICE output, GK_NORMALIZE, n_fit and row ranges; GK_DIST and row maps are
 * GK_ERR_UNSUPPORTED.  gk_rw_iterations copies the CG iterations / series terms of every entry of the last K
 * (rows x cols u8, row-major). */
#define GK_RW_CG 0
#define GK_RW_SPECTRAL 1
#define GK_RW_SERIES 2
#define GK_RW_FINITE 0
#define GK_RW_EXP 1
#define GK_RW_INV 2
#define GK_RW_LABELED 1 /* gk_rw_features flag: RandomWalkLabeled (the packed labels mask the product graph) */
int gk_rw_features(gk_handle* h, int32_t route, int32_t fn, double lamda, const double* coef, int32_t n_coef,
                   const double* values, const int32_t* t_row_ptr, const int32_t* t_col_idx, const double* t_values,
                   const double* q, const double* w, int32_t flags, gk_stats* stats);
int gk_rw_iterations(gk_handle* h, uint8_t* out);

/* SubgraphMatching (subgraph_matching.py), one graph pair per warp.  The packed CSR gives each graph's edges
 * (self-loops are ignored), the packed labels its vertex label ids, edge_label[E] the edge label ids of the packed
 * edges (with an edge kernel).  Vertex weights cv(a, b) are 1 (GK_SM_KV_NONE), [La == Lb] (GK_SM_KV_DIRAC) or
 * vtable[La * n_vlabels + Lb]; c-edge weights 1 (GK_SM_KE_NONE), [Lea == Leb] (GK_SM_KE_DIRAC) or
 * etable[Lea * n_elabels + Leb]; each table at most 4096 finite entries.  tv[s - 1] (s = 1 .. k; tv[k] = 0, and
 * k = 0 gives tv[0] = sum cv) sums the connected cliques of the weighted product graph; gk_gram (gram_path 13) returns
 * K = fma chain over lambdas[0 .. k] * tv from 0.  Integer-valued tables are summed exactly (a sum of 2^53 or more
 * is GK_ERR_RANGE), real ones in fp64.  Real lambdas with k + 1 > 15, and cliques past 32 vertices, are
 * GK_ERR_UNSUPPORTED.  gk_gram: fp64 only, host or GK_OUT_DEVICE output, GK_NORMALIZE, n_fit and row ranges; GK_DIST
 * and row maps are GK_ERR_UNSUPPORTED.  gk_sm_counts writes tv of the n_fit pairs of row `row` of the gk_gram
 * request with the same n_fit: out[n_fit * (k + 1)]. */
#define GK_SM_KV_NONE 1
#define GK_SM_KV_DIRAC 2
#define GK_SM_KE_NONE 4
#define GK_SM_KE_DIRAC 8
int gk_sm_features(gk_handle* h, int32_t k, const double* lambdas, const double* vtable, int32_t n_vlabels,
                   const double* etable, int32_t n_elabels, const int32_t* edge_label, int32_t flags, gk_stats* stats);
int gk_sm_counts(gk_handle* h, int64_t n_fit, int64_t row, double* out);

/* WeisfeilerLehman over SubgraphMatching (weisfeiler_lehman.py over subgraph_matching.py) in one clique enumeration.
 * level_ids[v * (n_iter + 1) + h] is the WL class of packed vertex v at level h (any numbering per level; level 0 is
 * the partition of the packed labels, and each level refines the one before).  The vertex kernel is GK_SM_KV_DIRAC
 * or GK_SM_KV_NONE (level_ids may then be null: every level has every product vertex); the edge kernel, the edge
 * labels, k and the lambdas are those of gk_sm_features, whose checks apply.  gk_gram then returns
 * K = ((K_0 + K_1) + K_2) ... in fp64, K_h the SubgraphMatching K of the level-h classes as vertex labels, under
 * gk_sm_features' gk_gram rules; GK_NORMALIZE divides by that sum's own self similarities.  (n_iter + 1) *
 * min(k, largest packed graph) above 64 is GK_ERR_UNSUPPORTED.  gk_sm_wl_counts writes tv of every level of the
 * n_fit pairs of row `row`: out[n_fit * (n_iter + 1) * (k + 1)], pair-major then level. */
int gk_sm_wl_features(gk_handle* h, int32_t k, int32_t n_iter, const int32_t* level_ids, const double* lambdas,
                      const double* etable, int32_t n_elabels, const int32_t* edge_label, int32_t flags,
                      gk_stats* stats);
int gk_sm_wl_counts(gk_handle* h, int64_t n_fit, int64_t row, double* out);

/* HadamardCode over SubgraphMatching (hadamard_code.py over subgraph_matching.py) in one clique enumeration.
 * level_ids[v * n_iter + h] is the HadamardCode class of packed vertex v at level h = 0 .. n_iter - 1 (any numbering
 * per level: only equality within a level is read; after gk_hc_features, gk_wl_labels returns the classes of each
 * level).  The levels need not refine each other.  The vertex kernel is GK_SM_KV_DIRAC (the level-h product graph has
 * the vertex pairs of equal level-h classes) or GK_SM_KV_NONE (level_ids may then be null: every level is the same);
 * the edge kernel, the edge labels, k and the lambdas are those of gk_sm_features, whose checks apply.  gk_gram then
 * returns K = ((K_0 + K_1) + K_2) ... in fp64, K_h the SubgraphMatching K of the level-h classes as vertex labels,
 * under gk_sm_features' gk_gram rules (GK_NORMALIZE, n_fit, row ranges, GK_OUT_DEVICE; no GK_DIST, no row map);
 * GK_NORMALIZE divides by that sum's own self similarities.  n_iter * min(k, largest packed graph) above 64 is
 * GK_ERR_UNSUPPORTED, before anything is launched. */
int gk_sm_hc_features(gk_handle* h, int32_t k, int32_t n_iter, const int32_t* level_ids, const double* lambdas,
                      const double* etable, int32_t n_elabels, const int32_t* edge_label, int32_t flags,
                      gk_stats* stats);

/* OddSth (odd_sth.py), one warp per root vertex.  The packed CSR lists every vertex's out-neighbours in the reference's
 * edge-dictionary order (every packed vertex is a root), the packed labels are one id per distinct str(label), and
 * rank[V] orders the label values within each graph (equal values share a rank).  Root v's DAG is the BFS from v cut
 * at depth h (h < 0: no limit), ordered by Kahn's algorithm with the (rank, insertion sequence) priority; every DAG
 * node's subtree identity is interned exactly (hash, verification of (label id, child identities), and a repeat with
 * another seed on a detected collision: stats->hash_retries).  phi[f, g] counts the (root, node) pairs of graph g with
 * identity f, and C[f] = phi[f, g0] for the first graph g0 that has f.  gk_gram (gram_path 14) returns
 * K[i, j] = sum_f C[f] phi[f, i] phi[f, j] exactly in fp64 (one exact integer Gram per bit of C, summed as
 * sum_b 2^b G_b), with K / sqrt(d_i d_j) under GK_NORMALIZE and xdiag / ydiag = d.  In a transform (n_fit < N) the
 * transformed graphs' identities take part in numbering and in d, as in the reference.  gk_gram: fp64 only, host or
 * GK_OUT_DEVICE output, GK_NORMALIZE, n_fit and row ranges; GK_DIST and row maps are GK_ERR_UNSUPPORTED.
 * GK_ERR_UNSUPPORTED also for a graph of more than 4096 vertices and for 2^30 or more (root, vertex) or (root, edge)
 * pairs (sum of n^2, sum of n m).  h == 0 is GK_ERR_ARG.  flags must be 0.  stats: n_columns = identities,
 * n_levels = bit planes of C, level_dims = columns per plane, n_entries = node slots (sum of n^2), hash_retries,
 * ms_hash (DAGs and identities), ms_columns.
 * gk_odd_info writes [identities, child ids of all signatures, largest C]; gk_odd_signatures the signature of every
 * identity (label[F], child_off[F + 1], child[child_off[F]] identity ids in order, C[F]). */
int gk_odd_features(gk_handle* h, int32_t depth, const int32_t* rank, int32_t flags, gk_stats* stats);
/* WeisfeilerLehman over OddSth: the pass of gk_odd_features over n_iter + 1 label sets at once.  ids and rank are
 * [n_iter + 1][V]: level l's label ids (non-negative, every id of level l above every id of level l - 1, so the
 * identities of different levels are disjoint) and rank values (non-negative).  Each level's DAGs take their own node
 * and child slots; one (graph, identity) table then holds the sum over the levels, and gk_gram (gram_path 14) returns
 * sum_levels K_level exactly.  The 4096-vertex and 2^30-pair limits apply to the (n_iter + 1)-fold totals and are
 * checked before anything is sized. */
int gk_wl_odd_features(gk_handle* h, int32_t depth, int32_t n_iter, const int32_t* ids, const int32_t* rank,
                       int32_t flags, gk_stats* stats);
int gk_odd_info(gk_handle* h, int64_t* info3);
int gk_odd_signatures(gk_handle* h, int32_t* label, int64_t* child_off, int32_t* child, int32_t* C);
/* Tests only: the next `attempts` identity passes of gk_odd_features hash (label id, number of children) alone, so
 * only the verification separates identities and every such pass must detect a collision and be repeated. */
int gk_selftest_odd_collision(gk_handle* h, int32_t attempts);

/* MultiscaleLaplacian (multiscale_laplacian.py), fp64 throughout, in stages because the reference's eigen-decompositions
 * of the sampled blocks run on the host between them.  The packed CSR (with weights) must be a symmetric adjacency
 * with non-negative weights and graphs of at most 128 vertices; gamma > 0 and heta > 0.  Every matrix is then SPD and
 * is factored by Cholesky; a non-positive pivot met anyway is GK_ERR_RANGE, never a NaN in K.
 *   gk_ml_begin    dense adjacency, the radius-l balls for l = 1 .. L (level 1 lists a vertex with a self-loop twice,
 *                  as the reference's [v] + neighbours(v)), and phi[V * dim] as the current features.  A non-symmetric
 *                  adjacency, L > 64, gamma or heta <= 0 and a graph of more than 128 vertices are GK_ERR_UNSUPPORTED.
 *                  stats: ms_h2d, ms_features (adjacency and balls).
 *   gk_ml_project  features <- features Q, Q[rows * cols] row-major with rows = the current width; the new width must
 *                  lie in [1, 32] (else GK_ERR_UNSUPPORTED).  stats: ms_combine.
 *   gk_ml_level    every vertex's record at `level` (1 .. L): S = U^T (L_nb + heta I)^-1 U + gamma I over its
 *                  neighbourhood nb, record = (S^-1 row-major, log det S), P' * P' + 1 doubles.  The level's sample
 *                  records are those of the vertices samples[ns] (fit: also written to samp_rec_out if given, and the
 *                  ns x ns block of the new features at those rows to K_samples if given) or samp_rec[ns] (transform).
 *                  The new features are K_proj[v, m] = flg(sample m, vertex v), V x ns, ns <= 1024 (else
 *                  GK_ERR_UNSUPPORTED).  stats: ms_features (records), ms_rw (projection), ms_d2h.
 *   gk_ml_finish   every packed graph's final record over its whole Laplacian, written to rec_out[N] if given; the
 *                  Gram's records are fit_rec[n_fit] (the fitted graphs' final records, 0 in a fit) followed by them.
 *                  stats: ms_features.
 * flg(a, b) = exp((-log det(S_a^-1 + S_b^-1) - (ld_a + ld_b) / 2) / 2), 0 when the exponent is below -30.
 * gk_gram (gram_path 15) returns K[r, c] = flg(record row_g0 + r, record c) over the records, one warp per pair: fp64
 * only, host or GK_OUT_DEVICE output, GK_NORMALIZE, n_fit and row ranges (n_fit counts records); the full square case
 * computes the upper triangle and mirrors it, and xdiag / ydiag come from the same pair function.  GK_DIST and row
 * maps are GK_ERR_UNSUPPORTED. */
int gk_ml_begin(gk_handle* h, int32_t L, double gamma, double heta, const double* phi, int32_t dim, gk_stats* stats);
int gk_ml_project(gk_handle* h, const double* Q, int32_t rows, int32_t cols, gk_stats* stats);
int gk_ml_level(gk_handle* h, int32_t level, const int32_t* samples, int32_t ns, const double* samp_rec,
                double* samp_rec_out, double* K_samples, gk_stats* stats);
int gk_ml_finish(gk_handle* h, const double* fit_rec, int64_t n_fit, double* rec_out, gk_stats* stats);

/* SvmTheta (svm_theta.py), fp64 throughout, per graph of 1 .. 128 vertices (more is GK_ERR_UNSUPPORTED).
 *   gk_svmt_solve  sizes[N] vertices per graph, adj[V * 4] the row-major 128-bit out-edge masks of every vertex
 *                  (bit j of row i: A[i][j] > 1e-10, diagonal cleared).  Launches, and returns without waiting for:
 *                  the smallest eigenvalue m of the mask with its upper triangle mirrored (scipy's eigvalsh with
 *                  lower=False), then libsvm's one-class SMO (nu = 0.5, tol = 1e-3, shrinking) on K = mask / -m with a
 *                  unit diagonal when m < -1e-6, else on the mask itself, with libsvm's float Q entries and its rounding
 *                  of every operation.  A solve that does not converge within 10^7 iterations is GK_ERR_RANGE in
 *                  gk_svmt_phi.  stats: n_graphs, n_vertices.
 *   gk_svmt_draw   host only: numpy's legacy `RandomState.choice(n, level, replace=False)` for every graph in order,
 *                  every level lo + li (li < n_levels) not above n in ascending order, counts[g * n_levels + li] times
 *                  each; appends the drawn indexes to idx[n_idx] (n_idx must be the schedule's total).  mt_key[624] /
 *                  mt_pos are the MT19937 state of `get_state()`, advanced in place.
 *   gk_svmt_phi    phi[g][li] = mean over the level's samples of the sum of the alphas at the drawn indexes (all n alphas
 *                  for a level above n), 0 without samples, both in numpy's summation order; idx / counts as given to
 *                  gk_svmt_draw.  A total index count other than the schedule's, or a drawn index not below its graph's
 *                  vertex count, is GK_ERR_ARG.  Optional outputs: phi[N * n_levels], m_out[N], alpha_out[V], iters_out[N].  The
 *                  first level of each graph follows fit_phi0[n_fit] (the fitted graphs', 0 in a fit) as the rows of
 *                  gk_gram.  stats: ms_h2d (both calls' uploads), ms_features (eigenvalues), ms_rw (SMO), ms_combine
 *                  (phi), ms_d2h.
 * gk_gram (gram_path 16) returns K[r][c] = phi0[row_g0 + r] * phi0[c], fp64 only, host or GK_OUT_DEVICE output,
 * GK_NORMALIZE (by sqrt(d_r d_c), d = phi0^2), n_fit and row ranges (n_fit counts rows).  GK_DIST and row maps are
 * GK_ERR_UNSUPPORTED. */
int gk_svmt_solve(gk_handle* h, int64_t n_graphs, const int32_t* sizes, const uint32_t* adj, gk_stats* stats);
int gk_svmt_draw(uint32_t* mt_key, int32_t* mt_pos, int64_t n_graphs, const int32_t* sizes, int32_t lo,
                 int32_t n_levels, const int32_t* counts, uint8_t* idx, int64_t n_idx);
int gk_svmt_phi(gk_handle* h, int32_t lo, int32_t n_levels, const int32_t* counts, const uint8_t* idx, int64_t n_idx,
                const double* fit_phi0, int64_t n_fit, double* phi, double* m_out, double* alpha_out, int32_t* iters_out,
                gk_stats* stats);

/* GraphletSampling, sampled route (graphlet_sampling.py:290-463, `sampling` a dict).  The packed CSR is each graph's
 * 0/1 adjacency (A > 0), rows ascending; labels are ignored.
 *   gk_gs_draw      host only: for every graph of `sizes` in order, n_samples times, r = rs.randint(min(3, n),
 *                   min(k, n) + 1) (no draw when the two are equal) and rs.choice(n, r, replace=False) on numpy's
 *                   legacy MT19937 stream (mt_key[624] / mt_pos of `get_state()`, advanced in place): samp_size[g *
 *                   n_samples + t] = r and the indexes appended to idx (n_idx of them, idx_cap >= n_samples * sum
 *                   min(k, n)).  k > 6 is GK_ERR_UNSUPPORTED.
 *   gk_gs_features  every sample of the graphs g0 .. N-1 (samp_off[N - g0 + 1] sample offsets, samp_size, idx as
 *                   gk_gs_draw wrote them) classified on the device: the class is the undirected sample graph (a pair
 *                   is an edge when either direction is, a diagonal entry a self-loop) up to isomorphism, exact for up
 *                   to 6 vertices.  prior[n_prior][3] = (graph < g0, class code, samples) restores the counts of an
 *                   earlier run (gk_gs_counts).  The first n_fit packed graphs are the fitted ones: a graph's count of
 *                   a class is its samples + 1 unless it is the first fitted graph with that class, or, for a class no
 *                   fitted graph has, the first new graph with it.  The arguments (offsets, sample sizes, index
 *                   count, prior rows, counts below 2^31) are checked before the first launch; a drawn index outside
 *                   its graph is found by the classification kernel, which skips that sample, and is GK_ERR_ARG with no
 *                   feature block left behind.  A self similarity of 2^53 or more is GK_ERR_RANGE.  gk_gram (gram_path
 *                   17, fp64 output only: a K entry above 2^24 would not be exact in fp32) then returns the exact
 *                   integer Gram, GK_NORMALIZE by self similarities over all classes.
 *                   stats: n_columns (classes), n_entries (samples), ms_hash (class table), ms_h2d, ms_features
 *                   (classification), ms_columns.
 *   gk_gs_counts    the table of the last gk_gs_features as rows (graph, class code, samples, count) sorted by graph
 *                   and code; *n_out is the row count, the rows are written when cap >= it. */
int gk_gs_draw(uint32_t* mt_key, int32_t* mt_pos, int64_t n_graphs, const int32_t* sizes, int32_t k, int64_t n_samples,
               uint8_t* samp_size, int32_t* idx, int64_t idx_cap, int64_t* n_idx);
int gk_gs_features(gk_handle* h, int32_t k, int64_t n_fit, int64_t g0, const int64_t* samp_off,
                   const uint8_t* samp_size, const int32_t* idx, int64_t n_idx, const int64_t* prior, int64_t n_prior,
                   gk_stats* stats);
int gk_gs_counts(gk_handle* h, int64_t cap, int64_t* out, int64_t* n_out);

/* Propagation / PropagationAttr (propagation.py:27-689).  The packed CSR (gk_pack_csr without weights; with the
 * label ids for the labelled kernel) is the sparsity pattern of every graph's row-normalised transition matrix T,
 * t_values[E] its entries.  P (V x dim, fp64) starts one-hot from the packed label ids or as p0[V * dim] (GK_PK_ATTR).
 * Level t = 0 .. t_max-1 hashes every vertex with u[t * dim ..] and b, then P <- T P (each entry one FMA chain over
 * the row's entries in ascending column order):
 *   labelled     bin = floor((dot(P_v, u_t) + b[t]) / w), sqrt(P) first with GK_PK_SQRT (M = "H")
 *   GK_PK_ATTR   bin = the dim-tuple floor((P_vj u_tj + b[t * dim + j]) / w); P is stored back rounded to float32
 *                (GK_PK_STORE_F32) or truncated toward zero (GK_PK_STORE_INT), as numpy's assignment into P does
 * GK_PK_NEW_LABELS (labels unseen at fit, propagation.py:328-395): the vertices of graphs >= n_fit that have a label
 * id >= dim_orig (level 0), or whose columns >= dim_orig are all positive (later levels), hash the full row with
 * u_t; every other vertex uses the columns < dim_orig.  Those private bins never equal a bin of another vertex kind,
 * and each of them also counts in the transformed graph before its own when it is that graph's successor's first
 * vertex (the reference's inclusive upper bound).  Without the flag dim_orig must equal dim.
 * Every level's bins become columns of their own and (graph, column) counts an SP-layout feature block: gk_gram's
 * integer route gives K = sum_t Phi_t Phi_t^T (fp32 / fp64, normalisation, n_fit, row ranges, GK_OUT_DEVICE); row maps
 * and GK_DIST are GK_ERR_UNSUPPORTED.  A NaN bin is GK_ERR_UNSUPPORTED; a P that does not fit is GK_ERR_RANGE.
 * stats: n_columns, ms_hash (propagate + hash), ms_propagate, ms_columns, pk_near_edge.  t_max in [1, 64], w != 0. */
#define GK_PK_ATTR 1
#define GK_PK_SQRT 2
#define GK_PK_STORE_F32 4
#define GK_PK_STORE_INT 8
#define GK_PK_NEW_LABELS 16
int gk_pk_features(gk_handle* h, int32_t t_max, double w, const double* u, const double* b, int32_t dim,
                   int32_t dim_orig, int64_t n_fit, const double* t_values, const double* p0, int32_t flags,
                   gk_stats* stats);
/* bins of level `level` after gk_pk_features: out[V * K] (K = dim for GK_PK_ATTR, else 1; -0.0 stored as 0.0), and
 * priv[V] (may be NULL) = 1 where the vertex hashed as a private (new-label) vertex */
int gk_pk_hashes(gk_handle* h, int32_t level, double* out, uint8_t* priv);

/* PyramidMatch (pyramid_match.py:18-285) and WeisfeilerLehman over it.  The vertex embeddings are made on the host
 * (the reference's eigs / numpy.linalg.eig calls, absolute values): U[n_sets * V * d] fp64, vertex v's row at
 * (s * V + v) * d, and n_cols[n_sets * N] the column count of every graph's embedding (min(n, d) on the eig branch);
 * entries past a graph's column count are ignored, and so is every vertex with skip[v] != 0 (skip[V] may be NULL: a
 * vertex of the packed block that the base kernel's graph does not contain).  Every used value must lie in
 * [0, 1 + 2^-(L-1)) -- the |U| of unit eigenvectors do -- else GK_ERR_ARG.  Level j < L puts every entry (v, q < n_cols) into cell
 * floor(u * 2^j) (2^j clamped to 2^j - 1) of histogram row label(v) * d + q:
 *   GK_PM_LABELS     label = the packed label id (one set)
 *   GK_PM_WL_LABELS  label = WL level s of the gk_wl_features(n_iter) call just before (n_sets = n_iter + 1)
 *   neither          row = q
 * Every (set, level) becomes a unary-expanded count block of its own (the NeighborhoodHash layout).  gk_gram then
 * returns, per set, the reference's fp64 combine of the level intersections I_j = sum min(cnt, cnt') replayed in its
 * order, summed over the sets in set order (gram_path 11): fp64 only, host or GK_OUT_DEVICE output, GK_NORMALIZE,
 * n_fit and row ranges; xdiag / ydiag are the same replay of I_j = n * n_cols (n without the skipped vertices).  GK_DIST and row maps are
 * GK_ERR_UNSUPPORTED, as are L > 64, V * d >= 2^31, d * (largest graph) >= 2^24 (fp32 counts) and keys whose row
 * << (L - 1) does not fit 64 bits.  stats: n_levels = n_sets * L blocks, level_dims = distinct cells per block,
 * n_columns, ms_columns.  gk_pm_cells writes the cell of every entry e = v * d + q of one set and level (-1 for
 * q >= n_cols or a skipped vertex): out[V * d]. */
#define GK_PM_LABELS 1
#define GK_PM_WL_LABELS 2
int gk_pm_features(gk_handle* h, int32_t n_iter, int32_t L, int32_t d, const double* U, const int32_t* n_cols,
                   const uint8_t* skip, int32_t n_sets, int32_t flags, gk_stats* stats);
int gk_pm_cells(gk_handle* h, int32_t set, int32_t level, int64_t* out);

/* HadamardCode (hadamard_code.py:24-391) over VertexHistogram or ShortestPath.  Every vertex carries a vector of
 * `width` (W, a power of two) int64 entries: at level 0 row `label` of Sylvester's Hadamard matrix,
 * H[r, c] = (-1)^popcount(r & c), for the packed label id r (< W: the reference's label enumeration); at level i >= 1
 * its own level-(i-1) vector plus those of its out-neighbours, wrapping modulo 2^64 like numpy's int64 additions.
 * Vertices with skip[v] != 0 (skip[V] may be NULL) are absent from the levels >= 1: labelled vertices that are not
 * keys of the reference's edge dictionary.  n_iter in [1, 64) levels (level 0 included).  Classes of a level are
 * exact vector equality (hashed, then verified vector by vector; a collision repeats the pass with another seed).
 *   flags 0          VertexHistogram: the (graph, level column) counts of every level in one FK_WL block, so gk_gram
 *                    returns the reference's sum of per-level matrices, with everything gk_gram supports for WL
 *   GK_HC_SP         ShortestPath(with_labels=True): the labelled path histogram of every level in one FK_SP block
 *                    (as gk_wl_sp_features); GK_SP_DIJKSTRA_ORDER selects the path-sum order of real weights.  No
 *                    vertex may be skipped.
 * GK_ERR_ARG for a packed label >= width, a width that is not a power of two or n_iter out of range;
 * GK_ERR_UNSUPPORTED when the two V x W x 8-byte level buffers do not fit in device memory.
 * stats: level_dims = classes per level, hash_retries, ms_hash = the relabel (vectors, classes, VH counts).
 * gk_hc_vectors recomputes the vectors of one level of the last gk_hc_features call on the packed block:
 * out[V * W], vertex v's vector at v * W (zeros for a skipped vertex at levels >= 1).
 * gk_selftest_hc_collision (tests only): the next gk_hc_features starts with a degenerate hash (every z_c = 0), so its
 * verification must see collisions and its retry must give the right classes.
 * gk_selftest_wl_collision (tests only): the next `attempts` WL relabel attempts on the handle -- each iteration of
 * gk_wl_features' retry loop, and the asynchronous pass of gk_wl_gram, counts as one -- hash every vertex of the levels
 * >= from_level by its own label and degree only, on every relabel route, so vertices with equal (label, degree) and
 * different neighbour labels share a hash slot and only the signature verification can tell their classes apart.
 * attempts > 8 exhausts gk_wl_features' retries. */
#define GK_HC_SP 8
int gk_hc_features(gk_handle* h, int32_t n_iter, int32_t width, const uint8_t* skip, int32_t flags, gk_stats* stats);
int gk_hc_vectors(gk_handle* h, int32_t level, int64_t* out);
int gk_selftest_hc_collision(gk_handle* h);
int gk_selftest_wl_collision(gk_handle* h, int32_t attempts, int32_t from_level);

/* Gram matrix of the current feature block.
 *   n_fit == n_graphs : K is [n_graphs x n_graphs]                      (fit_transform)
 *   n_fit <  n_graphs : K is [(n_graphs-n_fit) x n_fit], rows = Y graphs (transform)
 *   row_begin,row_end : only rows [row_begin,row_end) of K are computed and written
 *                       (multi-GPU row tiling); K_out points at row `row_begin`.
 *   K_out may be NULL (result stays on the device; see gk_fetch).
 *   xdiag[n_fit], ydiag[n_graphs-n_fit] : self-similarities (fp64, host) or NULL.      */
int gk_gram(gk_handle* h, int64_t n_fit, int32_t flags, int64_t row_begin, int64_t row_end,
            void* K_out, int32_t out_dtype, int64_t ld, double* xdiag, double* ydiag,
            gk_stats* stats);

/* Row map: packed graph g contributes to row row_of_graph[g] of K (n_rows rows in total; gk_gram's
 * n_fit / row ranges / diagonals then count rows).  Used by CoreFramework (core_framework.py:177-223):
 * the k-core subgraphs of every graph are packed as separate graphs with level-tagged labels (their
 * feature columns are therefore disjoint) and mapped back to their graph's row, so one Gram equals the
 * reference's scatter-add of one base-kernel matrix per core level.  Cleared by gk_pack_csr;
 * n_rows <= 0 restores the identity. */
int gk_set_row_map(gk_handle* h, int64_t n_rows, const int32_t* row_of_graph);

/* ---- multi-GPU: one process per GPU, one handle per process (SURVEY 8b/8e: the N x N output tiled over GPUs,
 * a final all-gather over NVLink only when the whole matrix must live on every device).
 * Every rank packs the same block and runs the same feature call (the relabel prologue is replicated: the whole
 * graph set is a few tens of MB); gk_gram with GK_DIST then computes the rank's row block [gk_comm_rows) of K.
 * The SYRK tiles are shared between the ranks -- each off-diagonal 256 x 256 tile is computed once, by one of
 * the two ranks that own its rows / columns -- and the GEMM epilogue stores the mirrored half straight into the
 * owning rank's row block through peer-mapped memory (CUDA IPC over NVLink), so the exchange overlaps the MMA
 * tile by tile and no rank recomputes what another one has.  NCCL carries the bootstrap, the handle exchange,
 * the two barriers of a call and, with GK_DIST_GATHER, the in-place all-gather of the finished row blocks
 * (BASELINE config 4: the full fp32 K on every rank, library-owned: gk_result_device / gk_fetch).
 * gk_comm_unique_id: rank 0 creates the 128-byte NCCL id, the application hands it to every rank (any channel).
 * All of these are collective: every rank calls them in the same order with the same sizes. */
#define GK_DIST 64          /* gk_gram flag: row block of this rank, tiles shared with the peers */
#define GK_DIST_GATHER 128  /* gk_gram flag: GK_DIST + all-gather, the full K stays on every device */
int gk_comm_unique_id(void* out128);
int gk_comm_init(gk_handle* h, int32_t nranks, int32_t rank, const void* unique_id128);
int gk_comm_destroy(gk_handle* h);  /* collective; gk_destroy calls it */
/* the row block of this rank: ceil(n_rows / nranks) rounded up to 256 rows per rank (identity without a communicator) */
int gk_comm_rows(gk_handle* h, int64_t n_rows, int64_t* row_begin, int64_t* row_end);
/* library-owned device result of the last gk_gram (valid until the next call on the handle) */
int gk_result_device(gk_handle* h, void** ptr, int64_t* rows, int64_t* cols, int64_t* ld, int32_t* dtype);
/* host-only (tests): the {row, column} tile list gk_gram(GK_DIST) gives rank `rank` of `nranks` */
int gk_selftest_dist_tiles(int64_t n_rows, int32_t nranks, int32_t rank, int32_t* tiles_xy, int64_t cap, int64_t* n_tiles);

/* Copy rows of the device-resident K of the last gk_gram to the host. */
int gk_fetch(gk_handle* h, void* K_out, int32_t out_dtype, int64_t ld);

/* WL inspection (parity tests): compressed label of every vertex at `level`
 * (dense ids, first-occurrence order) */
int gk_wl_labels(gk_handle* h, int32_t level, int32_t* out);

/* APSP matrix of graph g (n x n fp64, inf = unreachable): after gk_sp_features(GK_SP_KEEP_DIST), or after
 * gk_spattr_features -- the (S, phi) tuples of shortest_path.py:77-129 that ShortestPathAttr with a user `metric`
 * contracts pair by pair on the host (grakel/kernels/shortest_path.py:130-164, kernel.py:236-296) */
int gk_sp_distances(gk_handle* h, int64_t g, double* out);

/* WL features + square Gram of the packed block in ONE call: gk_wl_features followed by gk_gram(n_fit = N)
 * (weisfeiler_lehman.py:199-328 for fit_transform).  When the request is the plain square case with an fp32 device
 * result (flags 0 / GK_OUT_DEVICE / GK_DENSE_ALL; K_out NULL = library-owned, a device pointer, or a float64 host
 * matrix) the whole pass is enqueued without a host synchronisation in the middle: the head/tail threshold is chosen
 * on the device and the host sizes buffers by the capacities earlier passes left; anything that does not fit (first
 * call, hash collision, counts beyond the exact range) repeats through the two synchronous calls. */
int gk_wl_gram(gk_handle* h, int32_t n_iter, int32_t flags, void* K_out, int32_t out_dtype, int64_t ld,
               double* xdiag, gk_stats* stats);

/* One-call forms with host buffers (the e2e path that bench.py times). */
int gk_wl_fit_transform(gk_handle* h, int64_t n_graphs, const int32_t* graph_ptr,
                        const int32_t* row_ptr, const int32_t* col_idx, const int32_t* labels,
                        int32_t n_iter, int32_t flags, void* K_out, int32_t out_dtype, int64_t ld,
                        double* diag, gk_stats* stats);
int gk_sp_fit_transform(gk_handle* h, int64_t n_graphs, const int32_t* graph_ptr,
                        const int32_t* row_ptr, const int32_t* col_idx, const int32_t* labels,
                        const double* weights, int32_t sp_flags, int32_t flags, void* K_out,
                        int32_t out_dtype, int64_t ld, double* diag, gk_stats* stats);

/* ---- TU-format dataset files -> packed CSR block (host side; no device work).
 * Replaces grakel/datasets/base.py:135-290 (read_data: <name>_graph_indicator.txt, _A.txt, _node_labels.txt,
 * _node_attributes.txt, _edge_labels.txt, _graph_labels.txt parsed into per-graph Python sets and dicts) and
 * the per-graph Graph parsing that follows it (graph.py:147-230, 982-1053): the arrays gk_tu_fill writes are
 * exactly what gk_pack_csr takes.  Edge semantics as in read_data: an edge line belongs to the graph of its
 * source, GK_TU_SYMMETRIC adds the reverse edge (base.py:216-218), duplicates collapse, the last edge-label
 * line of a pair wins (:262-266). */
typedef struct gk_tu gk_tu;
#define GK_TU_SYMMETRIC 1      /* read_data(is_symmetric=True) */
#define GK_TU_ATTR_NODES 2     /* read_data(prefer_attr_nodes=True): node attributes instead of node labels */
#define GK_TU_DEGREE_LABELS 4  /* read_data(produce_labels_nodes=True) when there is no node-label file */
/* vertex set of the packed block */
#define GK_TU_LABELLED_NODES 0 /* every labelled node: what WeisfeilerLehman / VertexHistogram walk */
#define GK_TU_EDGE_NODES 1     /* nodes that occur in an edge: ShortestPath(+Attr) and WL-OA (edge-dictionary keys) */
int gk_tu_open(const char* dir, const char* name, int32_t flags, gk_tu** out);
/* info[0..7] = graphs, nodes, edge lines, has node labels, has edge labels, has classes, attribute dim, 0 */
int gk_tu_info(const gk_tu* t, int64_t* info);
/* choose the vertex set, build the CSR; returns the sizes of the arrays gk_tu_fill writes */
int gk_tu_pack(gk_tu* t, int32_t mode, int64_t* n_vertices, int64_t* n_edges);
/* graph_ptr[graphs+1], row_ptr[V+1], col_idx[E] (GLOBAL vertex ids, rows sorted), node_labels[V] (raw integer
 * labels), edge_labels[E], attrs[V*dim], classes[graphs], node_of_vertex[V] (1-based file node id); any may be NULL */
int gk_tu_fill(const gk_tu* t, int32_t* graph_ptr, int32_t* row_ptr, int32_t* col_idx, int32_t* node_labels,
               int32_t* edge_labels, double* attrs, int32_t* classes, int32_t* node_of_vertex);
int gk_tu_close(gk_tu* t);

/* CUDA-event timing on the handle's stream (bench.py). */
int gk_event_record(gk_handle* h, int32_t slot);            /* slot in [0,16) */
int gk_event_elapsed(gk_handle* h, int32_t a, int32_t b, float* ms);

/* cudaProfilerStart / cudaProfilerStop (on != 0 / on == 0): lets a profiler capture one
 * steady-state pass (tools/profile_step.py under `ncu --profile-from-start off`). */
int gk_profiler_range(int32_t on);

/* Self-test of the tensor-core Gram on a dense count matrix (tests only):
 * counts[n*d] (uint16), out_tc / out_simt [n*n] fp64. */
int gk_selftest_gram(gk_handle* h, int64_t n, int64_t d, const uint16_t* counts, double* out_tc,
                     double* out_simt);

/* Bytes of device memory and of pinned host memory the library's buffers hold right now, over every handle of the
 * process (tests only: a handle's create-use-destroy cycle must return both to where they were). */
int gk_selftest_live_bytes(int64_t* device, int64_t* pinned);

/* ---- float64 result buffers on the host (the reference returns a fresh float64 ndarray, kernel.py:167-204).
 * gk_host_alloc maps `bytes` of anonymous memory with transparent huge pages requested; gk_host_free returns
 * the block to a small per-process pool (GRAKEL_B200_HOST_POOL_MB, default 2048; 0 = unmap at once), so a loop
 * of fit_transform calls re-uses already-faulted pages.  The Python layer wraps the block in an ndarray whose
 * finaliser calls gk_host_free.  Any host pointer is accepted as K_out of gk_gram; these are just the fast ones. */
int gk_host_alloc(int64_t bytes, void** out);
int gk_host_free(void* p, int64_t bytes);

/* Host-only self test of the result delivery (tests only; no device needed): src[rows*cols] fp32 on the host
 * -> dst[rows*cols] fp64 through the same band / widen / mirror code gk_gram uses after its D2H copies.
 * mode 0: symmetric square, upper triangle only; 1: all rows; 2: all rows, normalised by diag (+ nan_to_num). */
int gk_selftest_deliver(int32_t mode, int64_t rows, int64_t cols, const float* src, const double* diag,
                        int32_t nan_to_num, double* dst);

#ifdef __cplusplus
}
#endif
#endif
