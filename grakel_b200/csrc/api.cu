// C-ABI of the grakel_b200 engine (see include/grakel_b200.h for the contract and
// the reference file:line each entry point replaces).  sm_90a (H100) only.
#include <algorithm>
#include <array>
#include <climits>
#include <cmath>
#include <cstdlib>
#include <condition_variable>
#include <functional>
#include <memory>
#include <mutex>
#include <atomic>
#include <thread>

#include <immintrin.h>
#include <pthread.h>
#include <sched.h>

#include <cuda_profiler_api.h>

#include "common.cuh"
#include "features.cuh"
#include "gram_tc.cuh"
#include "gram_tc2.cuh"
#include "sp.cuh"
#include "spattr.cuh"
#include "graph_hopper.cuh"
#include "wl.cuh"
#include "wl_fused2.cuh"
#include "wl_oa.cuh"
#include "neighborhood_hash.cuh"
#include "random_walk.cuh"
#include "propagation.cuh"
#include "pyramid_match.cuh"
#include "hadamard_code.cuh"
#include "nspd.cuh"
#include "subgraph_matching.cuh"
#include "odd_sth.cuh"
#include "multiscale_laplacian.cuh"
#include "svm_theta.cuh"
#include "graphlet_sampling.cuh"
#include "tu_reader.h"
#include "comm.h"

namespace gk {
thread_local std::string g_last_error;
std::atomic<int64_t> g_live_bytes[2] = {};

static inline size_t next_pow2(size_t x) {
  size_t p = 1;
  while (p < x) p <<= 1;
  return p;
}
static inline int cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

// Cost model of the head/tail split of the Gram: the dense rate of the GEMM per panel type (flop/s; measured on an
// H100 SXM at a 400 W power limit with every shared column dense: 7.8e14 bf16; 1.51e15 u8, 2.06x the bf16 rate of
// the same run, tools/bench_u8_gram.py) and the amortised cost of one pair update of K.
// The update cost is not a single measured figure: below ~32 updates per 32 x 32 block of K they ride in the GEMM
// epilogue almost for free, beyond it they overflow to global atomics into DRAM.  It is set so that the model's argmin
// matches sweeps of the forced threshold on the same card (GRAKEL_B200_FORCE_T, config 2, ms per pass):
//   bf16 panel: T = 8 / 16 / 32 / 64 / 128 / 256 -> 1.48 / 1.19 / 0.97 / 2.04 / 2.72 / 4.39; the model picks T = 32
//   u8 panel:   T = 8 / 16 / 32 / 64 / 128 / 256 -> 1.15 / 0.99 / 0.92 / 2.01 / 2.75 / 4.47; the model picks T = 32
//   (the forced passes zero the whole panel pitch; the model's own T = 32 pass runs in 0.83 ms)
// Halving the head's cost per column does not move the argmin: the tail's cost jumps by ~0.3 ms from T = 32 to 64
// (updates overflow the epilogue's lists), far more than the 0.09 ms of u8 MMAs the 1 279 extra head columns cost.
constexpr double COST_GEMM_RATE_BF16 = 7.8e14;
constexpr double COST_GEMM_RATE_U8 = 1.5e15;
constexpr double COST_T_ATOMIC = 6.7e-11;

// Element type of the integer head panel: u8 when every count is <= 255 (u8 x u8 -> s32 wgmma, twice the bf16 rate),
// else bf16 (exact up to 256).  GRAKEL_B200_U8=0 keeps bf16 everywhere (A/B switch).
static bool u8_panel_enabled() {
  const char* e = getenv("GRAKEL_B200_U8");
  return !(e && atoi(e) == 0);
}
static inline int panel_bk(int elem_bytes) { return elem_bytes == 1 ? BK_U8 : BK; }  // elements per 128-byte k-block
static inline double panel_rate(int elem_bytes) { return elem_bytes == 1 ? COST_GEMM_RATE_U8 : COST_GEMM_RATE_BF16; }

// cuTensorMapEncodeTiled through the runtime's driver entry point (no -lcuda)
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn get_encode() {
  static const EncodeTiledFn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    return cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
                   q == cudaDriverEntryPointSuccess
               ? reinterpret_cast<EncodeTiledFn>(p)
               : nullptr;
  }();
  return fn;
}

// integer head panel, `elem_bytes` 1 (u8) or 2 (bf16): one 128-byte swizzle row per k-block
static int make_panel_map(CUtensorMap* m, void* base, long long cols, long long rows, int box_rows, int elem_bytes) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return fail(GK_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)cols * elem_bytes};
  cuuint32_t box[2] = {(cuuint32_t)panel_bk(elem_bytes), (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(m, elem_bytes == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, base, dims,
                   strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(GK_ERR_CUDA, "cuTensorMapEncodeTiled failed: " + std::to_string((int)r));
  return GK_OK;
}

// fp32 (tf32 operand) panel: 32 elements = one 128-byte swizzle row per k-block
static int make_panel_map_f32(CUtensorMap* m, void* base, long long cols, long long rows, int box_rows) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return fail(GK_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)cols * 4};
  cuuint32_t box[2] = {(cuuint32_t)BK_TF32, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, base, dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(GK_ERR_CUDA, "cuTensorMapEncodeTiled(f32 panel) failed: " + std::to_string((int)r));
  return GK_OK;
}

// fp32 K as a 2-D tensor for TMA stores of 32x32 blocks (128-byte swizzle)
static int make_out_map(CUtensorMap* m, void* base, long long cols, long long rows, long long ld) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return fail(GK_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 4};
  cuuint32_t box[2] = {32, 32};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(GK_ERR_CUDA, "cuTensorMapEncodeTiled(out) failed: " + std::to_string((int)r));
  return GK_OK;
}

static int read_scalars(gk_handle* h, DevScalars** out) {
  GK_TRY(h->h_scalars.ensure(sizeof(DevScalars)));
  GK_CUDA(cudaMemcpyAsync(h->h_scalars.p, h->scalars.p, sizeof(DevScalars), cudaMemcpyDeviceToHost, h->stream));
  GK_CUDA(cudaStreamSynchronize(h->stream));
  *out = h->h_scalars.as<DevScalars>();
  return GK_OK;
}

static float ev_ms(cudaEvent_t a, cudaEvent_t b) {
  float ms = 0.f;
  cudaEventElapsedTime(&ms, a, b);
  return ms;
}

}  // namespace gk

using namespace gk;

#define LAUNCH_CHECK(h)                                 \
  do {                                                  \
    (h)->launches++;                                    \
    GK_CUDA(cudaGetLastError());                        \
  } while (0)

// The entry check of a call on the packed block.  It selects the handle's device, which some argument checks query.
static int need_packed(gk_handle* h, const char* who) {
  if (!h) return fail(GK_ERR_ARG, "null handle");
  if (h->N <= 0) return fail(GK_ERR_STATE, std::string(who) + ": no graphs packed");
  GK_CUDA(cudaSetDevice(h->dev));
  return GK_OK;
}

// A feature pass calls features_begin after its argument checks, before it writes any handle state, and
// features_publish as its last state change.  A refused call leaves the previous block; a failed pass leaves none.
static void features_begin(gk_handle* h) {
  h->feature_kind = FK_NONE;
  h->pro_ready = false;
}

static void features_publish(gk_handle* h, FeatureKind kind) { h->feature_kind = kind; }

extern "C" {

int gk_version(void) { return 100; }
const char* gk_last_error(void) { return g_last_error.c_str(); }

int gk_create(int device_ordinal, gk_handle** out) {
  if (!out) return fail(GK_ERR_ARG, "gk_create: out is NULL");
  int n = 0;
  GK_CUDA(cudaGetDeviceCount(&n));
  if (device_ordinal < 0 || device_ordinal >= n) return fail(GK_ERR_ARG, "gk_create: bad device ordinal");
  GK_CUDA(cudaSetDevice(device_ordinal));
  cudaDeviceProp prop;
  GK_CUDA(cudaGetDeviceProperties(&prop, device_ordinal));
  if (prop.major != 9 || prop.minor != 0) {
    return fail(GK_ERR_UNSUPPORTED, std::string("grakel_b200 needs an sm_90a (H100) device, found sm_") +
                                        std::to_string(prop.major) + std::to_string(prop.minor));
  }
  std::unique_ptr<gk_handle> h(new gk_handle());
  h->dev = device_ordinal;
  h->sm_count = prop.multiProcessorCount;
  GK_CUDA(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
  GK_CUDA(cudaStreamCreateWithFlags(&h->stream2, cudaStreamNonBlocking));
  GK_CUDA(cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming));
  GK_CUDA(cudaEventCreateWithFlags(&h->ev_join, cudaEventDisableTiming));
  for (auto& e : h->ev_stage) GK_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  for (auto& e : h->ev) GK_CUDA(cudaEventCreate(&e));
  for (auto& e : h->tev) GK_CUDA(cudaEventCreate(&e));
  GK_TRY(h->scalars.ensure(sizeof(DevScalars)));
  GK_TRY(h->h_scalars.ensure(sizeof(DevScalars)));
  GK_CUDA(cudaFuncSetAttribute(gram_tc_kernel<float, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, GEMM_SMEM));
  GK_CUDA(cudaFuncSetAttribute(gram_tc_kernel<double, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, GEMM_SMEM));
  GK_CUDA(cudaFuncSetAttribute(gram_tc_kernel<float, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, GEMM_SMEM));
  GK_CUDA(cudaFuncSetAttribute(gram_tc_kernel<double, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, GEMM_SMEM));
  GK_CUDA(cudaFuncSetAttribute(gram_tc_kernel<float, false, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, GEMM_SMEM));
  GK_CUDA(cudaFuncSetAttribute(gram_tc_kernel<double, false, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, GEMM_SMEM));
  GK_CUDA(cudaFuncSetAttribute(gram_tc_kernel<float, true, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, GEMM_SMEM));
  GK_CUDA(cudaFuncSetAttribute(gram_tc_kernel<double, true, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, GEMM_SMEM));
  GK_CUDA(cudaFuncSetAttribute(gram_tc2_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, GEMM2_SMEM));
  GK_CUDA(cudaFuncSetAttribute(gram_tc2_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, GEMM2_SMEM));
  GK_CUDA(cudaFuncSetAttribute(gram_tc_kernel<double, false, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, GEMM_SMEM));
  GK_CUDA(cudaFuncSetAttribute(wl_fused2_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, WLF2_SMEM));
  GK_CUDA(cudaFuncSetAttribute(wl_fused2_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, WLF2_SMEM));
  *out = h.release();
  return GK_OK;
}

// --------------------------------------------------------------------------- multi-GPU (comm.h)
int gk_comm_unique_id(void* out128) {
  if (!out128) return fail(GK_ERR_ARG, "gk_comm_unique_id: null argument");
  NcclApi* api = nccl_api();
  if (!api->lib || !api->error.empty()) return fail(GK_ERR_UNSUPPORTED, "gk_comm_unique_id: " + api->error);
  static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
  ncclUniqueId id;
  GK_NCCL(api, api->GetUniqueId(&id));
  memcpy(out128, &id, sizeof(id));
  return GK_OK;
}

int gk_comm_destroy(gk_handle* h) {
  if (!h || !h->comm) return GK_OK;
  Comm* c = reinterpret_cast<Comm*>(h->comm);
  cudaSetDevice(h->dev);
  cudaStreamSynchronize(h->stream);
  for (int r = 0; r < c->nranks; ++r)
    if (r != c->rank && c->peer_base[r]) { cudaIpcCloseMemHandle(c->peer_base[r]); c->peer_base[r] = nullptr; }
  // collective: nobody frees an exported block (~gk_handle does, right after this) before every peer has unmapped it
  if (c->comm && c->nranks > 1 && nccl_api()->AllReduce) {
    nccl_api()->AllReduce(c->d_token, c->d_token, 1, ncclInt32, ncclSum, c->comm, h->stream);
    cudaStreamSynchronize(h->stream);
  }
  if (c->d_token) cudaFree(c->d_token);
  if (c->d_handles) cudaFree(c->d_handles);
  NcclApi* api = nccl_api();
  if (c->comm && api->CommDestroy) api->CommDestroy(c->comm);
  delete c;
  h->comm = nullptr;
  return GK_OK;
}

int gk_comm_init(gk_handle* h, int32_t nranks, int32_t rank, const void* unique_id128) {
  if (!h || !unique_id128) return fail(GK_ERR_ARG, "gk_comm_init: null argument");
  if (nranks < 1 || nranks > DIST_MAX_RANKS || rank < 0 || rank >= nranks) return fail(GK_ERR_ARG, "gk_comm_init: 1..8 ranks");
  if (h->comm) return fail(GK_ERR_STATE, "gk_comm_init: the handle already has a communicator");
  NcclApi* api = nccl_api();
  if (!api->lib || !api->error.empty()) return fail(GK_ERR_UNSUPPORTED, "gk_comm_init: " + api->error);
  GK_CUDA(cudaSetDevice(h->dev));
  Comm* c = new Comm();
  c->nranks = nranks; c->rank = rank;
  ncclUniqueId id;
  memcpy(&id, unique_id128, sizeof(id));
  ncclResult_t r = api->CommInitRank(&c->comm, nranks, id, rank);
  if (r != ncclSuccess) { delete c; return fail(GK_ERR_CUDA, std::string("ncclCommInitRank: ") + api->GetErrorString(r)); }
  if (cudaMalloc(&c->d_token, 256) != cudaSuccess || cudaMalloc(&c->d_handles, (size_t)(nranks + 1) * 64) != cudaSuccess) {
    delete c;
    return fail(GK_ERR_CUDA, "gk_comm_init: cudaMalloc failed");
  }
  cudaMemset(c->d_token, 0, 256);
  h->comm = c;
  return GK_OK;
}

int gk_comm_rows(gk_handle* h, int64_t n_rows, int64_t* row_begin, int64_t* row_end) {
  if (!h || !row_begin || !row_end || n_rows < 0) return fail(GK_ERR_ARG, "gk_comm_rows: bad arguments");
  Comm* c = reinterpret_cast<Comm*>(h->comm);
  const int nranks = c ? c->nranks : 1, rank = c ? c->rank : 0;
  const long long per = dist_rows_per_rank(n_rows, nranks);
  *row_begin = std::min<long long>(n_rows, rank * per);
  *row_end = std::min<long long>(n_rows, (rank + 1) * per);
  return GK_OK;
}

// Host-only: the tile list of one rank (tests of the partition; no device, no communicator needed)
int gk_selftest_dist_tiles(int64_t n_rows, int32_t nranks, int32_t rank, int32_t* tiles_xy, int64_t cap, int64_t* n_tiles) {
  if (!n_tiles || nranks < 1 || nranks > DIST_MAX_RANKS || rank < 0 || rank >= nranks) return fail(GK_ERR_ARG, "gk_selftest_dist_tiles: bad arguments");
  std::vector<int2> t;
  dist_tiles(n_rows, nranks, rank, t);
  *n_tiles = (int64_t)t.size();
  if (tiles_xy)
    for (size_t i = 0; i < t.size() && (int64_t)i < cap; ++i) { tiles_xy[2 * i] = t[i].x; tiles_xy[2 * i + 1] = t[i].y; }
  return GK_OK;
}

int gk_destroy(gk_handle* h) {
  if (h) delete h;
  return GK_OK;
}

int gk_sync(gk_handle* h) {
  if (!h) return fail(GK_ERR_ARG, "null handle");
  GK_CUDA(cudaStreamSynchronize(h->stream));
  return GK_OK;
}

int gk_event_record(gk_handle* h, int32_t slot) {
  if (!h || slot < 0 || slot >= 16) return fail(GK_ERR_ARG, "gk_event_record: bad slot");
  GK_CUDA(cudaEventRecord(h->ev[slot], h->stream));
  return GK_OK;
}
int gk_event_elapsed(gk_handle* h, int32_t a, int32_t b, float* ms) {
  if (!h || !ms || a < 0 || a >= 16 || b < 0 || b >= 16) return fail(GK_ERR_ARG, "gk_event_elapsed: bad args");
  GK_CUDA(cudaEventSynchronize(h->ev[b]));
  GK_CUDA(cudaEventElapsedTime(ms, h->ev[a], h->ev[b]));
  return GK_OK;
}

// ncu/nsys capture range (tools/profile_step.py runs under `--profile-from-start off`)
int gk_profiler_range(int32_t on) {
  GK_CUDA(on ? cudaProfilerStart() : cudaProfilerStop());
  return GK_OK;
}

// ---------------------------------------------------------------------------
int gk_pack_csr(gk_handle* h, int64_t n_graphs, const int32_t* graph_ptr, const int32_t* row_ptr,
                const int32_t* col_idx, const int32_t* labels, const double* weights, const double* attrs,
                int32_t attr_dim) {
  if (!h) return fail(GK_ERR_ARG, "null handle");
  if (n_graphs <= 0 || !graph_ptr || !row_ptr) return fail(GK_ERR_ARG, "gk_pack_csr: empty input");
  if (n_graphs >= (1LL << 31) - 1) return fail(GK_ERR_ARG, "gk_pack_csr: too many graphs");
  GK_CUDA(cudaSetDevice(h->dev));
  const int64_t N = n_graphs;
  const int64_t V = graph_ptr[N];
  if (graph_ptr[0] != 0 || V < 0) return fail(GK_ERR_ARG, "gk_pack_csr: bad graph_ptr");
  if (V >= (1LL << 26)) return fail(GK_ERR_ARG, "gk_pack_csr: more than 2^26 vertices in one block");
  const int64_t E = V ? row_ptr[V] : 0;
  if (E < 0 || (E > 0 && !col_idx)) return fail(GK_ERR_ARG, "gk_pack_csr: bad row_ptr / col_idx");
  // graph sizes (N small); every per-vertex / per-edge scan runs on the device below
  int max_n = 0;
  for (int64_t g = 0; g < N; ++g) {
    const int n = graph_ptr[g + 1] - graph_ptr[g];
    if (n < 0 || graph_ptr[g + 1] > V) return fail(GK_ERR_ARG, "gk_pack_csr: graph_ptr not monotone");
    max_n = std::max(max_n, n);
  }
  features_begin(h);  // a new block starts without features
  h->N = N; h->V = V; h->E = E;
  h->has_weights = weights != nullptr;
  h->has_labels = labels != nullptr;
  h->attr_dim = attrs ? attr_dim : 0;
  h->max_graph_size = max_n;
  h->n_rows = 0;  // ... without a row map
  h->hc_W = 0;    // ... and without HadamardCode vectors
  h->ml_w = 0;    // ... and without MultiscaleLaplacian features
  h->wl_tiles_valid = false;
  h->graph_ptr_host.assign(graph_ptr, graph_ptr + N + 1);
  h->graph_eptr_host.resize(N + 1);
  for (int64_t g = 0; g <= N; ++g) h->graph_eptr_host[g] = V ? row_ptr[graph_ptr[g]] : 0;

  GK_CUDA(cudaEventRecord(h->tev[0], h->stream));
  GK_TRY(h->graph_ptr.ensure((N + 1) * 4));
  GK_TRY(h->row_ptr.ensure((V + 1) * 4));
  GK_TRY(h->col_idx.ensure(std::max<int64_t>(E, 1) * 4));
  GK_TRY(h->vgraph.ensure(std::max<int64_t>(V, 1) * 4));
  GK_TRY(h->large_list.ensure(std::max<int64_t>(V, 1) * 4 + 64));
  GK_CUDA(cudaMemcpyAsync(h->graph_ptr.p, graph_ptr, (N + 1) * 4, cudaMemcpyHostToDevice, h->stream));
  GK_CUDA(cudaMemcpyAsync(h->row_ptr.p, row_ptr, (V + 1) * 4, cudaMemcpyHostToDevice, h->stream));
  if (E) GK_CUDA(cudaMemcpyAsync(h->col_idx.p, col_idx, E * 4, cudaMemcpyHostToDevice, h->stream));
  if (labels) {
    GK_TRY(h->labels0.ensure(std::max<int64_t>(V, 1) * 4));
    GK_CUDA(cudaMemcpyAsync(h->labels0.p, labels, V * 4, cudaMemcpyHostToDevice, h->stream));
  }
  if (weights && E) {
    GK_TRY(h->weights.ensure(E * 8));
    GK_CUDA(cudaMemcpyAsync(h->weights.p, weights, E * 8, cudaMemcpyHostToDevice, h->stream));
  }
  if (attrs && attr_dim > 0) {
    GK_TRY(h->attrs.ensure((size_t)V * attr_dim * 8));
    GK_CUDA(cudaMemcpyAsync(h->attrs.p, attrs, (size_t)V * attr_dim * 8, cudaMemcpyHostToDevice, h->stream));
  }
  // device-side statistics + validation (degree histogram, bounds, labels, weights)
  int* d_scan = reinterpret_cast<int*>(h->scalars.as<DevScalars>()) ;  // reuse the scalar block as 16 ints
  GK_CUDA(cudaMemsetAsync(d_scan, 0, 64, h->stream));
  int hscan[16] = {0};
  if (V) {
    fill_vgraph<<<cdiv(V, 256), 256, 0, h->stream>>>((int)V, (int)N, h->graph_ptr.as<int>(), h->vgraph.as<int>());
    LAUNCH_CHECK(h);
    pack_scan<<<cdiv(V, 256), 256, 0, h->stream>>>((int)V, (int)E, h->graph_ptr.as<int>(), h->vgraph.as<int>(),
                                                   h->row_ptr.as<int>(), h->col_idx.as<int>(),
                                                   labels ? h->labels0.as<int>() : nullptr, d_scan);
    LAUNCH_CHECK(h);
    if (weights && E) {
      pack_scan_weights<<<h->sm_count * 4, 256, 0, h->stream>>>(E, h->weights.as<double>(), d_scan);
      LAUNCH_CHECK(h);
    }
    GK_CUDA(cudaMemcpyAsync(h->h_scalars.p, d_scan, 64, cudaMemcpyDeviceToHost, h->stream));
    GK_CUDA(cudaStreamSynchronize(h->stream));
    memcpy(hscan, h->h_scalars.p, 64);
  }
  if (hscan[6] & 1) return fail(GK_ERR_ARG, "gk_pack_csr: row_ptr not monotone");
  if (hscan[6] & 2) return fail(GK_ERR_ARG, "gk_pack_csr: edge leaves its graph");
  if (hscan[6] & 4) return fail(GK_ERR_ARG, "gk_pack_csr: negative label id");
  if (hscan[8] & 2) return fail(GK_ERR_UNSUPPORTED, "gk_pack_csr: negative or NaN edge weight");
  h->n_labels0 = labels ? hscan[7] + 1 : 0;
  h->unit_weights = !(hscan[8] & 1);
  h->max_degree = hscan[5];
  // WL signature kernel choice: one thread per vertex for degree <= 8 (cost ~1 lane), else
  // 16 or 32 lanes per vertex; vertices above the width take the warp-per-vertex kernel.
  {
    const long long above8 = (long long)hscan[2] + hscan[3] + hscan[4], above16 = (long long)hscan[3] + hscan[4],
                    above32 = hscan[4];
    const long long c8 = (long long)V * 1 + above8 * 32, c16 = (long long)V * 16 + above16 * 32,
                    c32 = (long long)V * 32 + above32 * 32;
    h->group_width = 8;
    h->n_large = above8;
    long long best = c8;
    if (c16 < best) { best = c16; h->group_width = 16; h->n_large = above16; }
    if (c32 < best) { best = c32; h->group_width = 32; h->n_large = above32; }
  }
  if (h->n_large) {
    GK_CUDA(cudaMemsetAsync(d_scan, 0, 4, h->stream));
    pack_large_list<<<cdiv(V, 256), 256, 0, h->stream>>>((int)V, h->row_ptr.as<int>(), h->group_width,
                                                         h->large_list.as<int>(), d_scan);
    LAUNCH_CHECK(h);
  }
  GK_CUDA(cudaEventRecord(h->tev[1], h->stream));
  GK_CUDA(cudaStreamSynchronize(h->stream));  // caller buffers may be reused once we return
  return GK_OK;
}

// ---------------------------------------------------------------------------
}  // extern "C"

template <int G>
static void launch_sig_small(gk_handle* h, const int* lab_in, unsigned long long seed, int degen) {
  const long long threads = (long long)h->V * G;
  wl_sig_small<G><<<cdiv(threads, 256), 256, 0, h->stream>>>(
      (int)h->V, h->row_ptr.as<int>(), h->col_idx.as<int>(), lab_in, h->sig_nbr.as<int>(), seed, degen,
      h->ht_keys.as<unsigned long long>(), h->ht_rep.as<int>(), (unsigned)(h->ht_cap - 1), h->slot_of.as<int>());
}

// (re)allocate and clear the statistics the feature kernels maintain at insert time
static int reset_feature_stats(gk_handle* h, int64_t col_cap, int64_t n_part, FeatStats* st, bool clear = true) {
  col_cap = std::max<int64_t>(col_cap, 1);
  n_part = std::max<int64_t>(n_part, 1);
  GK_TRY(h->part_max.ensure(n_part * 4));
  GK_TRY(h->part_new.ensure(n_part * 4));
  h->n_part = n_part;
  if (clear) {
    GK_CUDA(cudaMemsetAsync(h->part_max.p, 0, n_part * 4, h->stream));
    GK_CUDA(cudaMemsetAsync(h->part_new.p, 0, n_part * 4, h->stream));
  }
  st->part_max = h->part_max.as<unsigned>();
  st->part_new = h->part_new.as<unsigned>();
  GK_TRY(h->colcnt.ensure(col_cap * 4));
  GK_TRY(h->diag_u64.ensure(h->N * 8));
  h->col_cap = col_cap;
  if (clear) {
    GK_CUDA(cudaMemsetAsync(h->colcnt.p, 0, col_cap * 4, h->stream));
    GK_CUDA(cudaMemsetAsync(h->diag_u64.p, 0, h->N * 8, h->stream));
  }
  st->colcnt = h->colcnt.as<unsigned>();
  st->diag = h->diag_u64.as<unsigned long long>();
  st->sc = h->scalars.as<DevScalars>();
  return GK_OK;
}

static int init_scalars(gk_handle* h, int n_labels0) {
  DevScalars* hs = h->h_scalars.as<DevScalars>();
  memset(hs, 0, sizeof(DevScalars));
  hs->level_dims[0] = n_labels0;
  hs->level_base[0] = 0;
  hs->level_base[1] = n_labels0;
  GK_CUDA(cudaMemcpyAsync(h->scalars.p, hs, sizeof(DevScalars), cudaMemcpyHostToDevice, h->stream));
  // the pinned struct is reused for read-back; make sure the upload has consumed it
  GK_CUDA(cudaStreamSynchronize(h->stream));
  return GK_OK;
}

// gk_selftest_wl_collision: the level from which this relabel attempt hashes (own label, degree) only, INT_MAX for a
// normal attempt.  Every attempt (each iteration of gk_wl_features' retry loop, the asynchronous pass) takes one.
static int wl_take_degen(gk_handle* h) {
  if (h->wl_degen_attempts <= 0) return INT_MAX;
  --h->wl_degen_attempts;
  return h->wl_degen_from;
}

// What gk_wl_features decides and allocates before its first launch (shared with the asynchronous pass, gk_wl_gram)
struct WlPlan {
  int L = 0, G = 0, nb = 0, n_tiles = 0;
  bool fused = false;
  size_t ft_level_cap = 0;
};

static int wl_setup(gk_handle* h, int n_iter, WlPlan* pl) {
  const int64_t V = h->V, E = h->E;
  const int L = n_iter + 1;
  GK_TRY(h->labels_all.ensure((size_t)L * V * 4));
  GK_TRY(h->sig_nbr.ensure(std::max<int64_t>(E, 1) * 4 * 2));  // wl_fused2 double-buffers the rows by level parity
  GK_TRY(h->slot_of.ensure(V * 4));
  GK_TRY(h->flags.ensure(V * 4));
  const int nb = cdiv(V, 256);
  GK_TRY(h->block_sums.ensure((size_t)nb * 4));
  // >= 2 V slots (load <= 0.5 at the one level where almost every vertex is a class of its own; frozen vertices stop
  // inserting after it): three rotating tables stay L2-resident for the vertex counts of the benchmark workloads.
  h->ht_cap = std::max<size_t>(next_pow2((size_t)V * 2), 1024);
  GK_TRY(h->ht_keys.ensure(h->ht_cap * 8 * 3));  // three tables: the fused kernel rotates them over the levels
  GK_TRY(h->ht_rep.ensure(h->ht_cap * 4 * 2));
  const size_t ft_level_cap = std::max<size_t>(next_pow2((size_t)V * 2), 1024);  // one L2-sized sub-table per level
  // Fused persistent kernel (wl_fused2.cuh) whenever the graphs can be cut into shared-memory tiles of
  // whole graphs; otherwise (a graph above the tile capacity) the multi-kernel path below.
  bool fused = true;
  if (const char* e = getenv("GRAKEL_B200_WL_FUSED")) fused = atoi(e) != 0;
  const int G = std::min(h->sm_count, 1024);
  int n_tiles = 0;
  long long tiles_env = 0;
  if (const char* e = getenv("GRAKEL_B200_WL_TILES_PER_CTA")) tiles_env = atoi(e);
  if (fused && h->wl_tiles_valid && h->wl_tiles_key == tiles_env) {
    // same packed block as the last call: the partition is still in wlf_buf (the kernels only touch its barrier word)
    fused = h->wl_tiles_fused;
    n_tiles = h->wl_n_tiles;
  } else if (fused) {
    std::vector<int> tv, ct(G + 1, 0);
    bool ok = false;
    int64_t per0 = std::max<int64_t>(1, std::max((V + (int64_t)G * WLF_TILE_V - 1) / ((int64_t)G * WLF_TILE_V),
                                                  (E + (int64_t)G * WLF_TILE_E - 1) / ((int64_t)G * WLF_TILE_E)));
    if (const char* e = getenv("GRAKEL_B200_WL_TILES_PER_CTA")) per0 = std::max<int64_t>(per0, atoi(e));  // tests: multi-tile CTAs on small inputs
    for (int per = (int)per0;
         per <= 4096 && !ok; per *= 2) {
      // G * per tiles of whole graphs, balanced by vertex count
      const int T = G * per;
      tv.assign(T + 1, 0);
      size_t g = 0;
      for (int t = 1; t < T; ++t) {
        const long long want = (long long)V * t / T;
        while (g < (size_t)h->N && h->graph_ptr_host[g] < want) ++g;
        tv[t] = (int)g;
      }
      tv[T] = (int)h->N;
      ok = true;
      for (int t = 0; t < T && ok; ++t) {
        const int nv = h->graph_ptr_host[tv[t + 1]] - h->graph_ptr_host[tv[t]];
        const int ne = h->graph_eptr_host[tv[t + 1]] - h->graph_eptr_host[tv[t]];
        if (nv > WLF_TILE_V || ne > WLF_TILE_E) ok = false;
      }
      if (ok) {
        n_tiles = T;
        for (int t = 0; t <= T; ++t) tv[t] = h->graph_ptr_host[tv[t]];  // graph index -> first vertex
        for (int c = 0; c <= G; ++c) ct[c] = c * per;
        long long max_cta = 0;
        for (int c = 0; c < G; ++c) max_cta = std::max<long long>(max_cta, tv[ct[c + 1]] - tv[ct[c]]);
        if (max_cta >= WLF_CTA_V_LIMIT) ok = false;
      }
      if (h->max_graph_size > WLF_TILE_V) break;
    }
    fused = ok;
    if (fused) {
      // layout of wlf_buf (ints): [tile_vbeg (T+1) | cta_tile (G+1) | barrier]
      const size_t n_int = (size_t)(n_tiles + 1) + (G + 1) + 1;
      GK_TRY(h->wlf_buf.ensure(n_int * 4));
      GK_TRY(h->h_tiles.ensure(((size_t)n_tiles + G + 2) * 4));
      int* hp = h->h_tiles.as<int>();
      memcpy(hp, tv.data(), (size_t)(n_tiles + 1) * 4);
      memcpy(hp + n_tiles + 1, ct.data(), (size_t)(G + 1) * 4);
      GK_CUDA(cudaMemcpyAsync(h->wlf_buf.p, hp, ((size_t)n_tiles + G + 2) * 4, cudaMemcpyHostToDevice, h->stream));
    }
    h->wl_tiles_valid = true; h->wl_tiles_fused = fused; h->wl_n_tiles = n_tiles; h->wl_tiles_key = tiles_env;
  }
  // feature block: the multi-kernel path fills one open-addressing sub-table per level, the fused
  // kernel appends at most V entries per level to the same arrays used as a COO list
  h->ft_cap = fused ? std::max<size_t>((size_t)V * L, 1) : ft_level_cap * (size_t)L;
  if (h->ft_cap > (1ULL << 31)) return fail(GK_ERR_ARG, "gk_wl_features: feature table too large");
  GK_TRY(h->ft_keys.ensure(h->ft_cap * 8));
  GK_TRY(h->ft_cnt.ensure(h->ft_cap * 4));
  pl->L = L; pl->G = G; pl->nb = nb; pl->n_tiles = n_tiles; pl->fused = fused; pl->ft_level_cap = ft_level_cap;
  return GK_OK;
}

// prepare + wl_fused2 on the handle's stream; no synchronisation
static int wl_launch_v2(gk_handle* h, const WlPlan& pl, unsigned long long seed, int degen_from, const FeatStats& fst,
                        bool prof) {
  const int64_t V = h->V, E = h->E;
  const int L = pl.L, G = pl.G, n_tiles = pl.n_tiles;
  DevScalars* sc = h->scalars.as<DevScalars>();
  int* labels_all = h->labels_all.as<int>();
  {
      // wl_fused2.cuh: labels = representative vertex ids (one grid barrier per level), frozen singleton classes
      int* wb = h->wlf_buf.as<int>();
      int* d_cta_tile = wb + n_tiles + 1;
      unsigned* d_barrier = reinterpret_cast<unsigned*>(d_cta_tile + G + 1);
      GK_TRY(h->wl_single.ensure((size_t)V + 16));
      GK_TRY(h->diag_frozen.ensure((size_t)h->N * 8));
      {  // one launch clears everything the kernel expects cleared (no host upload, no synchronisation)
        Wlf2Prepare q;
        q.sc = sc; q.n_labels0 = h->n_labels0;
        q.part_max = h->part_max.as<unsigned>(); q.part_new = h->part_new.as<unsigned>(); q.n_part = h->n_part;
        q.colcnt = h->colcnt.as<unsigned>(); q.col_cap = h->col_cap;
        q.diag = h->diag_u64.as<unsigned long long>(); q.diag_frozen = h->diag_frozen.as<unsigned long long>(); q.n_graphs = h->N;
        q.barrier = d_barrier;
        q.frozen = h->wl_single.as<unsigned char>(); q.V = V;
        q.table1 = L > 1 ? h->ht_keys.as<unsigned long long>() + h->ht_cap : nullptr; q.ht_cap = (long long)h->ht_cap;
        wlf2_prepare_kernel<<<h->sm_count * 2, 1024, 0, h->stream>>>(q);
        LAUNCH_CHECK(h);
      }
      WlFused2Params fp;
      memset(&fp, 0, sizeof(fp));
      fp.V = (int)V; fp.L = L; fp.n_labels0 = h->n_labels0;
      fp.graph_ptr = h->graph_ptr.as<int>();
      fp.row_ptr = h->row_ptr.as<int>(); fp.col_idx = h->col_idx.as<int>(); fp.vgraph = h->vgraph.as<int>();
      fp.labels0 = h->labels0.as<int>(); fp.tile_vbeg = wb; fp.cta_tile = d_cta_tile;
      fp.barrier = d_barrier;
      fp.labels_all = labels_all; fp.sig_nbr = h->sig_nbr.as<int>(); fp.slot_of = h->slot_of.as<int>();
      fp.E = std::max<int64_t>(E, 1);
      {  // slot payloads (wl_fused2.cuh [A3]/[B]); GRAKEL_B200_WL_PAYLOAD=0: verify against the representative's CSR row
        const char* e = getenv("GRAKEL_B200_WL_PAYLOAD");
        if (!(e && atoi(e) == 0)) {
          GK_TRY(h->wl_payload.ensure(h->ht_cap * 32 * 2));
          fp.payload = h->wl_payload.as<int>();
        }
      }
      fp.frozen = h->wl_single.as<unsigned char>();
      fp.table = h->ht_keys.as<unsigned long long>();
      fp.ht_mask = (unsigned)(h->ht_cap - 1);
      fp.coo_keys = h->ft_keys.as<unsigned long long>(); fp.coo_cnt = h->ft_cnt.as<unsigned>();
      fp.seed = seed; fp.degen_from = degen_from; fp.st = fst; fp.sc = sc;
      fp.diag_frozen = h->diag_frozen.as<unsigned long long>();
      if (prof) {
        GK_TRY(h->K_stage.ensure((size_t)G * L * 128));
        GK_CUDA(cudaMemsetAsync(h->K_stage.p, 0, (size_t)G * L * 128, h->stream));
        fp.prof = h->K_stage.as<long long>();
      }
      void* args[] = {&fp};
      GK_CUDA(cudaLaunchCooperativeKernel(fp.payload ? (void*)wl_fused2_kernel<true> : (void*)wl_fused2_kernel<false>, dim3(G), dim3(WLF_THREADS), args, WLF2_SMEM, h->stream));
      LAUNCH_CHECK(h);
  }
  return GK_OK;
}

extern "C" {

int gk_wl_features(gk_handle* h, int32_t n_iter, gk_stats* stats) {
  GK_TRY(need_packed(h, "gk_wl_features"));
  if (!h->has_labels || h->V == 0) return fail(GK_ERR_ARG, "gk_wl_features: vertex labels are required");
  if (n_iter < 0 || n_iter + 1 >= MAX_LEVELS) return fail(GK_ERR_ARG, "gk_wl_features: n_iter out of range");
  const int64_t V = h->V, E = h->E;
  const int L = n_iter + 1;
  features_begin(h);
  h->n_levels = L;
  const int64_t launches0 = h->launches;

  WlPlan pl;
  GK_TRY(wl_setup(h, n_iter, &pl));
  const bool fused = pl.fused;
  const int G = pl.G, nb = pl.nb;
  const size_t ft_level_cap = pl.ft_level_cap;

  DevScalars* sc = h->scalars.as<DevScalars>();
  int* labels_all = h->labels_all.as<int>();
  int retries = 0;
  bool pro_enqueued = false;
  GK_CUDA(cudaEventRecord(h->tev[2], h->stream));
  for (;; ++retries) {
    pro_enqueued = false;
    if (retries > 8)
      return fail(GK_ERR_STATE, "gk_wl_features: repeated hash collisions (level mask 0x" +
                                    [&] { char b[16]; snprintf(b, sizeof(b), "%x", h->h_scalars.as<DevScalars>()->collision); return std::string(b); }() + ")");
    const unsigned long long seed = mix64(0x5851F42D4C957F2DULL + 0x9E3779B97F4A7C15ULL * (unsigned long long)retries);
    const int degen_from = wl_take_degen(h);
    FeatStats fst;
    if (!fused) GK_TRY(init_scalars(h, h->n_labels0));
    GK_TRY(reset_feature_stats(h, (int64_t)h->n_labels0 + V * (int64_t)(L - 1) + 1, (int64_t)std::max(nb, G) * L, &fst, !fused));
    h->wl_sparse_ids = false;
    if (fused) {
      const bool prof = getenv("GRAKEL_B200_PROF") != nullptr;
      GK_TRY(wl_launch_v2(h, pl, seed, degen_from, fst, prof));
      h->wl_sparse_ids = L > 1;
      GK_CUDA(cudaEventRecord(h->tev[3], h->stream));  // end of the feature stage
      if (!prof) {
        // Gram prologue of the square (fit_transform) case, enqueued BEFORE this call's one host synchronisation:
        // self similarities + per-CTA partials (diag_finish) and the column histogram (col_hist).  gk_gram then
        // finds everything its host-side decisions need (threshold T, D_c, exactness bounds) already on the host
        // and launches without a synchronisation of its own (pro_ready).
        const int64_t D = (int64_t)h->n_labels0 + V * (int64_t)(L - 1);
        GK_TRY(h->diag_f64.ensure(h->N * 8));
        GK_TRY(h->colstats.ensure(sizeof(ColStats)));
        GK_TRY(h->h_colstats.ensure(sizeof(ColStats)));
        diag_finish<<<cdiv(h->N, 256), 256, 0, h->stream>>>((int)h->N, h->diag_u64.as<unsigned long long>(), h->diag_f64.as<double>(),
                                                            (int)h->n_part, h->part_max.as<unsigned>(), h->part_new.as<unsigned>(), sc);
        LAUNCH_CHECK(h);
        GK_CUDA(cudaMemsetAsync(h->colstats.p, 0, sizeof(ColStats), h->stream));
        col_hist<<<cdiv(std::max<int64_t>(D, 1), 256), 256, 0, h->stream>>>(std::max<int64_t>(D, 1), 1, (int)h->N, h->colcnt.as<unsigned>(),
                                                                          nullptr, nullptr, h->colstats.as<ColStats>());
        LAUNCH_CHECK(h);
        GK_CUDA(cudaMemcpyAsync(h->h_colstats.p, h->colstats.p, sizeof(ColStats), cudaMemcpyDeviceToHost, h->stream));
        pro_enqueued = true;
      }
      if (prof) {  // raw int64 globaltimer stamps [G][L][16] (tools/prof_wl_phases.py)
        std::vector<long long> pr((size_t)G * L * 16);
        GK_CUDA(cudaMemcpyAsync(pr.data(), h->K_stage.p, pr.size() * 8, cudaMemcpyDeviceToHost, h->stream));
        GK_CUDA(cudaStreamSynchronize(h->stream));
        if (const char* out = getenv("GRAKEL_B200_PROF_OUT")) {
          if (FILE* f = fopen(out, "wb")) { fwrite(pr.data(), 8, pr.size(), f); fclose(f); }
        }
      }
    } else {
    GK_CUDA(cudaMemsetAsync(h->ft_keys.p, 0xFF, h->ft_cap * 8, h->stream));
    GK_CUDA(cudaMemsetAsync(h->ft_cnt.p, 0, h->ft_cap * 4, h->stream));
    GK_CUDA(cudaMemcpyAsync(labels_all, h->labels0.p, V * 4, cudaMemcpyDeviceToDevice, h->stream));
    wl_insert_level0<<<nb, 256, 0, h->stream>>>((int)V, labels_all, h->vgraph.as<int>(),
                                                 h->ft_keys.as<unsigned long long>(), h->ft_cnt.as<unsigned>(),
                                                 (unsigned)(ft_level_cap - 1), fst);
    LAUNCH_CHECK(h);
    for (int lv = 1; lv < L; ++lv) {
      const int* lab_in = labels_all + (size_t)(lv - 1) * V;
      int* lab_out = labels_all + (size_t)lv * V;
      const int degen = lv >= degen_from ? 1 : 0;
      GK_CUDA(cudaMemsetAsync(h->ht_keys.p, 0xFF, h->ht_cap * 8, h->stream));
      GK_CUDA(cudaMemsetAsync(h->ht_rep.p, 0x7F, h->ht_cap * 4, h->stream));
      if (h->group_width <= 8) {
        wl_sig_thread8<<<nb, 256, 0, h->stream>>>((int)V, h->row_ptr.as<int>(), h->col_idx.as<int>(), lab_in,
                                                  h->sig_nbr.as<int>(), seed, degen, h->ht_keys.as<unsigned long long>(),
                                                  h->ht_rep.as<int>(), (unsigned)(h->ht_cap - 1), h->slot_of.as<int>());
      } else if (h->group_width == 16) {
        launch_sig_small<16>(h, lab_in, seed, degen);
      } else {
        launch_sig_small<32>(h, lab_in, seed, degen);
      }
      LAUNCH_CHECK(h);
      if (h->n_large) {
        wl_sig_large<<<cdiv(h->n_large * 32, 256), 256, 0, h->stream>>>(
            (int)h->n_large, h->large_list.as<int>(), h->row_ptr.as<int>(), h->col_idx.as<int>(), lab_in,
            h->sig_nbr.as<int>(), seed, degen, h->ht_keys.as<unsigned long long>(), h->ht_rep.as<int>(),
            (unsigned)(h->ht_cap - 1), h->slot_of.as<int>());
        LAUNCH_CHECK(h);
      }
      wl_resolve<<<nb, 256, 0, h->stream>>>((int)V, h->row_ptr.as<int>(), lab_in, h->sig_nbr.as<int>(),
                                            h->ht_rep.as<int>(), h->slot_of.as<int>(), h->flags.as<int>(),
                                            h->block_sums.as<int>(), sc);
      LAUNCH_CHECK(h);
      wl_assign<<<nb, 256, 0, h->stream>>>((int)V, lv, h->flags.as<int>(), h->block_sums.as<int>(), lab_out, sc);
      LAUNCH_CHECK(h);
      wl_gather_insert<<<nb, 256, 0, h->stream>>>((int)V, lv, h->slot_of.as<int>(), lab_out, h->vgraph.as<int>(),
                                                   fst, h->ft_keys.as<unsigned long long>(),
                                                   h->ft_cnt.as<unsigned>(), (unsigned)(ft_level_cap - 1));
      LAUNCH_CHECK(h);
    }
    }  // multi-kernel path
    DevScalars* hs;
    GK_TRY(read_scalars(h, &hs));
    if (hs->ft_overflow) return fail(GK_ERR_STATE, "gk_wl_features: feature table overflow");
    if (!hs->collision) break;
  }
  if (!fused) {  // (wl_fused2 recorded the end of its stage right after the kernel; read_scalars synchronised)
    GK_CUDA(cudaEventRecord(h->tev[3], h->stream));
    GK_CUDA(cudaEventSynchronize(h->tev[3]));
  }
  DevScalars* hs = h->h_scalars.as<DevScalars>();
  h->n_columns = hs->level_base[L];
  if (pro_enqueued) {
    h->pro_hist = *h->h_colstats.as<ColStats>();
    h->pro_max_count = (long long)hs->max_count; h->pro_max_diag = (long long)hs->max_diag; h->pro_n_entries = (long long)hs->n_entries;
    h->pro_ready = true;
  }
  features_publish(h, FK_WL);
  if (stats) {
    memset(stats, 0, sizeof(*stats));
    stats->n_graphs = h->N; stats->n_vertices = V; stats->n_edges = E;
    stats->n_levels = L;
    for (int i = 0; i < L; ++i) stats->level_dims[i] = hs->level_dims[i];
    stats->n_columns = h->n_columns;
    if (h->wl_sparse_ids) {  // the column space is sparse (n_labels0 + (L-1) V wide); report the number of classes
      stats->n_columns = 0;
      for (int i = 0; i < L; ++i) stats->n_columns += hs->level_dims[i];
    }
    stats->hash_retries = retries;
    stats->kernel_launches = h->launches - launches0;
    stats->ms_features = ev_ms(h->tev[2], h->tev[3]);
  }
  return GK_OK;
}

// WL-OA: the WL feature block, then its unary expansion (wl_oa.cuh); one gk_gram of the expanded
// block is the histogram-intersection matrix of weisfeiler_lehman_optimal_assignment.py:257-266.
int gk_wl_oa_features(gk_handle* h, int32_t n_iter, gk_stats* stats) {
  gk_stats local;
  gk_stats* st = stats ? stats : &local;
  GK_TRY(gk_wl_features(h, n_iter, st));
  features_begin(h);
  const int64_t launches0 = h->launches;
  const int64_t D = std::max<int64_t>(h->n_columns, 1);
  const size_t out_cap = std::max<size_t>((size_t)h->V * (size_t)h->n_levels, 1);  // one entry per (vertex, level)
  if (out_cap > (1ULL << 31)) return fail(GK_ERR_ARG, "gk_wl_oa_features: feature block too large");
  GK_TRY(h->oa_keys.ensure(out_cap * 8));
  GK_TRY(h->oa_cnt.ensure(out_cap * 4));
  GK_TRY(h->oa_colcnt.ensure((out_cap + 1) * 4));
  GK_TRY(h->colmin.ensure(D * 4));  // scratch until the next gk_gram: largest count / first threshold column
  GK_TRY(h->colmax.ensure(D * 4));
  GK_TRY(h->colstats.ensure(std::max(sizeof(ColStats), sizeof(OaCursors))));
  GK_TRY(h->h_colstats.ensure(std::max(sizeof(ColStats), sizeof(OaCursors))));
  OaCursors* cur = h->colstats.as<OaCursors>();
  unsigned* colmaxcnt = h->colmin.as<unsigned>();
  unsigned* colbase = h->colmax.as<unsigned>();
  GK_CUDA(cudaMemsetAsync(cur, 0, sizeof(OaCursors), h->stream));
  GK_CUDA(cudaMemsetAsync(colmaxcnt, 0, D * 4, h->stream));
  GK_CUDA(cudaMemsetAsync(h->oa_keys.p, 0xFF, out_cap * 8, h->stream));
  GK_CUDA(cudaMemsetAsync(h->oa_colcnt.p, 0, (out_cap + 1) * 4, h->stream));
  GK_CUDA(cudaMemsetAsync(h->diag_u64.p, 0, h->N * 8, h->stream));
  oa_colmax<<<h->sm_count * 8, 256, 0, h->stream>>>(h->ft_cap, h->ft_keys.as<unsigned long long>(), h->ft_cnt.as<unsigned>(),
                                                    colmaxcnt);
  LAUNCH_CHECK(h);
  oa_colbase<<<cdiv(D, OA_THREADS), OA_THREADS, 0, h->stream>>>(D, colmaxcnt, colbase, cur);
  LAUNCH_CHECK(h);
  oa_expand<<<cdiv((long long)h->ft_cap, OA_THREADS), OA_THREADS, 0, h->stream>>>(
      h->ft_cap, h->ft_keys.as<unsigned long long>(), h->ft_cnt.as<unsigned>(), colbase, out_cap,
      h->oa_keys.as<unsigned long long>(), h->oa_cnt.as<unsigned>(), cur, h->oa_colcnt.as<unsigned>(),
      h->diag_u64.as<unsigned long long>(), h->scalars.as<DevScalars>());
  LAUNCH_CHECK(h);
  if (h->wl_sparse_ids) {  // frozen vertices wrote no entries: their (level) units of self similarity are kept aside
    add_u64<<<cdiv(h->N, 256), 256, 0, h->stream>>>((int)h->N, h->diag_frozen.as<unsigned long long>(), h->diag_u64.as<unsigned long long>());
    LAUNCH_CHECK(h);
  }
  h->n_part = 1;
  oa_finish<<<1, 1, 0, h->stream>>>(cur, h->part_max.as<unsigned>(), h->part_new.as<unsigned>(), h->scalars.as<DevScalars>(),
                                    h->wl_sparse_ids ? 1 : 0);
  LAUNCH_CHECK(h);
  GK_CUDA(cudaMemcpyAsync(h->h_colstats.p, cur, sizeof(OaCursors), cudaMemcpyDeviceToHost, h->stream));
  DevScalars* hs;
  GK_TRY(read_scalars(h, &hs));
  GK_CUDA(cudaEventRecord(h->tev[3], h->stream));
  GK_CUDA(cudaEventSynchronize(h->tev[3]));
  if (hs->ft_overflow) return fail(GK_ERR_STATE, "gk_wl_oa_features: expanded feature block overflow");
  const OaCursors hc = *h->h_colstats.as<OaCursors>();
  std::swap(h->ft_keys, h->oa_keys);
  std::swap(h->ft_cnt, h->oa_cnt);
  std::swap(h->colcnt, h->oa_colcnt);
  h->ft_cap = out_cap;
  h->col_cap = (int64_t)out_cap + 1;
  h->n_columns = (int64_t)hc.n_cols;
  features_publish(h, FK_WL);
  st->n_columns = h->n_columns;
  st->kernel_launches += h->launches - launches0;
  st->ms_features = ev_ms(h->tev[2], h->tev[3]);
  return GK_OK;
}

// dense first-occurrence ids of level `level` (>= 1) of a wl_fused2 run into `dst` (device, V ints)
static int wl_densify(gk_handle* h, int level, int* dst) {
  const int V = (int)h->V;
  const int nb = cdiv(V, DENS_THREADS);
  GK_TRY(h->block_sums.ensure((size_t)nb * 4));
  GK_TRY(h->flags.ensure((size_t)V * 4));
  const int* lab = h->labels_all.as<int>() + (size_t)level * V;
  wl_dens_count<<<nb, DENS_THREADS, 0, h->stream>>>(V, lab, h->block_sums.as<int>());
  LAUNCH_CHECK(h);
  wl_dens_scan<<<1, DENS_THREADS, 0, h->stream>>>(nb, h->block_sums.as<int>());
  LAUNCH_CHECK(h);
  wl_dens_rank<<<nb, DENS_THREADS, 0, h->stream>>>(V, lab, h->block_sums.as<int>(), h->flags.as<int>());
  LAUNCH_CHECK(h);
  wl_dens_apply<<<cdiv(V, 256), 256, 0, h->stream>>>(V, lab, h->flags.as<int>(), dst);
  LAUNCH_CHECK(h);
  return GK_OK;
}

int gk_wl_labels(gk_handle* h, int32_t level, int32_t* out) {
  if (!h || !out) return fail(GK_ERR_ARG, "gk_wl_labels: null argument");
  if (h->feature_kind != FK_WL || level < 0 || level >= h->n_levels) return fail(GK_ERR_STATE, "gk_wl_labels: no such level");
  GK_CUDA(cudaSetDevice(h->dev));
  const int* src = h->labels_all.as<int>() + (size_t)level * h->V;
  if (h->wl_sparse_ids && level >= 1) {
    GK_TRY(wl_densify(h, level, h->slot_of.as<int>()));
    src = h->slot_of.as<int>();
  }
  GK_CUDA(cudaMemcpyAsync(out, src, h->V * 4, cudaMemcpyDeviceToHost, h->stream));
  GK_CUDA(cudaStreamSynchronize(h->stream));
  return GK_OK;
}

// ---------------------------------------------------------------------------
// Shortest-path features.  Without a level label source: the ShortestPath kernel on the packed labels.
// With one (WeisfeilerLehman or HadamardCode over ShortestPath): the graphs were relabelled first, and the labelled
// path histogram of EVERY level goes into one feature block: label ids are made level-unique (id + first column of
// the level), so the levels use disjoint columns and one Gram equals the reference's sum of per-level matrices
// (weisfeiler_lehman.py:260-270, hadamard_code.py:217-236, with shortest_path.py:370-410 as the base kernel).
struct SpLabels {
  int n_pass = 1;
  const int* labels = nullptr;            // [n_pass][V] dense label ids of every level; null = the packed labels
  std::vector<long long> level_base{0};   // first label id of each level (n_pass + 1 entries)
};

static int sp_check(gk_handle* h, int32_t flags) {
  GK_TRY(need_packed(h, "gk_sp_features"));
  if ((flags & GK_SP_WITH_LABELS) && !h->has_labels) return fail(GK_ERR_ARG, "gk_sp_features: vertex labels are required");
  return GK_OK;
}

static int sp_features_impl(gk_handle* h, int32_t flags, const SpLabels& lab, gk_stats* stats) {
  const bool with_labels = flags & GK_SP_WITH_LABELS;
  const std::vector<long long>& level_base = lab.level_base;
  const int n_pass = lab.n_pass;
  const long long n_labels_total = lab.labels ? level_base[n_pass] : h->n_labels0;
  if (with_labels && n_labels_total >= (1 << 20)) return fail(GK_ERR_UNSUPPORTED, "gk_sp_features: more than 2^20 distinct labels");
  const bool use_u16 = (!h->has_weights || h->unit_weights) && h->max_graph_size < 16000;
  const size_t esz = use_u16 ? 2 : 8;
  const int64_t N = h->N;
  const int64_t launches0 = h->launches;
  features_begin(h);
  h->sp_flags = flags;

  // plan: graphs whose distance matrix fits the shared-memory budget vs the rest
  const size_t SMEM_DIST_MAX = 160 * 1024;
  std::vector<int> small, big;
  std::vector<int> bfs[4];  // unit weights: bitmask BFS with W = 1, 2, 4, 8 words (n <= 64 W)
  size_t max_small_nn = 0;
  h->sp_goff.assign(N + 1, 0);
  const bool keep = flags & GK_SP_KEEP_DIST;
  long long off_big = 0, off_all = 0;
  std::vector<long long> goff_big(N, 0);
  for (int64_t g = 0; g < N; ++g) {
    const long long n = h->graph_ptr_host[g + 1] - h->graph_ptr_host[g];
    h->sp_goff[g] = off_all;
    off_all += n * n;
    if (use_u16 && n <= 512) {
      bfs[n <= 64 ? 0 : n <= 128 ? 1 : n <= 256 ? 2 : 3].push_back((int)g);
    } else if ((size_t)(n * n) * esz <= SMEM_DIST_MAX) {
      small.push_back((int)g);
      max_small_nn = std::max(max_small_nn, (size_t)(n * n));
    } else {
      big.push_back((int)g);
      goff_big[g] = off_big;
      off_big += n * n;
    }
  }
  h->sp_goff[N] = off_all;
  const size_t smem_small = SP_LOCAL_SLOTS * 12 + max_small_nn * esz + 16;
  const size_t smem_big = SP_LOCAL_SLOTS * 12 + 16;

  // device buffers
  gk::DevBuf& lists = h->sp_lists;  // [small list | big list | BFS classes]
  GK_TRY(lists.ensure((size_t)N * 4 + 16));
  std::vector<int> order(small);
  order.insert(order.end(), big.begin(), big.end());
  size_t bfs_off[4];
  for (int i = 0; i < 4; ++i) { bfs_off[i] = order.size(); order.insert(order.end(), bfs[i].begin(), bfs[i].end()); }
  GK_CUDA(cudaMemcpyAsync(lists.p, order.data(), order.size() * 4, cudaMemcpyHostToDevice, h->stream));
  GK_TRY(h->sp_graph_off.ensure((size_t)(N + 1) * 8 * 2));
  long long* d_goff_all = h->sp_graph_off.as<long long>();
  long long* d_goff_big = d_goff_all + (N + 1);
  GK_CUDA(cudaMemcpyAsync(d_goff_all, h->sp_goff.data(), (N + 1) * 8, cudaMemcpyHostToDevice, h->stream));
  GK_CUDA(cudaMemcpyAsync(d_goff_big, goff_big.data(), N * 8, cudaMemcpyHostToDevice, h->stream));
  if (off_big) GK_TRY(h->sp_dist.ensure((size_t)off_big * esz));
  double* d_keep = nullptr;
  if (keep) {
    GK_TRY(h->K_stage.ensure((size_t)off_all * 8));
    d_keep = h->K_stage.as<double>();
  }
  GK_CUDA(cudaStreamSynchronize(h->stream));  // host vectors above go out of scope on retry

  if (use_u16) {
    GK_CUDA(cudaFuncSetAttribute(sp_apsp_hist<unsigned short>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max(smem_small, smem_big)));
  } else {
    GK_CUDA(cudaFuncSetAttribute(sp_apsp_hist<double>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max(smem_small, smem_big)));
  }

  size_t dict_cap = std::max<size_t>(h->sp_dict_cap, 1 << 16);
  // distance dictionary of real mode: its slot is the 24-bit distance field of a feature key, so it holds at most
  // 2^24 lengths (GRAKEL_B200_SP_DKEY_CAP=<slots> lowers the starting size, so that tests reach the regrowth)
  const size_t DKEY_CAP_MAX = (size_t)1 << 24;
  size_t dkey_cap = (size_t)1 << 18;
  if (const char* e = getenv("GRAKEL_B200_SP_DKEY_CAP"))
    dkey_cap = std::min(DKEY_CAP_MAX, next_pow2(std::max<size_t>(16, strtoull(e, nullptr, 10))));
  bool real_mode = false;
  size_t ft_cap = std::max<size_t>(next_pow2((size_t)std::max<int64_t>(h->V, 1024) * 16 * (size_t)std::min(n_pass, 4)), 1 << 20);
  DevScalars* sc = h->scalars.as<DevScalars>();
  GK_CUDA(cudaEventRecord(h->tev[2], h->stream));
  for (int attempt = 0;; ++attempt) {
    if (attempt > 6) return fail(GK_ERR_STATE, "gk_sp_features: tables keep overflowing");
    if (dict_cap > (1ULL << 28) || ft_cap > (1ULL << 31)) return fail(GK_ERR_STATE, "gk_sp_features: feature tables too large");
    GK_TRY(h->sp_dict_keys.ensure(dict_cap * 8));
    GK_TRY(h->ft_keys.ensure(ft_cap * 8));
    GK_TRY(h->ft_cnt.ensure(ft_cap * 4));
    h->sp_dict_cap = dict_cap;
    h->ft_cap = ft_cap;
    GK_TRY(init_scalars(h, 0));
    FeatStats fst;
    GK_TRY(reset_feature_stats(h, (int64_t)dict_cap, N, &fst));
    GK_CUDA(cudaMemsetAsync(h->sp_dict_keys.p, 0xFF, dict_cap * 8, h->stream));
    GK_CUDA(cudaMemsetAsync(h->ft_keys.p, 0xFF, ft_cap * 8, h->stream));
    GK_CUDA(cudaMemsetAsync(h->ft_cnt.p, 0, ft_cap * 4, h->stream));
    SpParams p;
    memset(&p, 0, sizeof(p));
    p.graph_ptr = h->graph_ptr.as<int>();
    p.row_ptr = h->row_ptr.as<int>();
    p.col_idx = h->col_idx.as<int>();
    p.weights = (h->has_weights && !use_u16) ? h->weights.as<double>() : nullptr;
    p.labels = with_labels ? h->labels0.as<int>() : nullptr;
    p.n_labels = with_labels ? (int)std::max<long long>(n_labels_total, 1) : 1;
    p.keep = d_keep;
    p.dict_keys = h->sp_dict_keys.as<unsigned long long>();
    p.dict_mask = (unsigned)(dict_cap - 1);
    p.ft_keys = h->ft_keys.as<unsigned long long>();
    p.ft_cnt = h->ft_cnt.as<unsigned>();
    p.ft_mask = (unsigned)(ft_cap - 1);
    p.sc = sc;
    p.st = fst;
    p.gdist = h->sp_dist.p;
    for (int pass = 0; pass < n_pass; ++pass) {
    if (lab.labels) {
      p.labels = lab.labels + (size_t)pass * h->V;
      p.label_offset = (int)level_base[pass];
    }
    if (real_mode) {
      // non-integer path lengths: (1) fp64 Floyd-Warshall of every graph into global memory + a
      // dictionary of the distinct distance bit patterns, (2) histogram keyed by (lu, lv, id(d))
      GK_TRY(h->sp_dist.ensure((size_t)std::max<long long>(off_all, 1) * 8));
      GK_TRY(h->sp_dkeys.ensure(dkey_cap * 8));
      GK_CUDA(cudaMemsetAsync(h->sp_dkeys.p, 0xFF, dkey_cap * 8, h->stream));
      SpParams pa = p;
      pa.gdist = h->sp_dist.p;
      pa.goff = d_goff_all;
      pa.dict_keys = h->sp_dkeys.as<unsigned long long>();
      pa.dict_mask = (unsigned)(dkey_cap - 1);
      pa.keep = nullptr;
      const size_t smem_a = max_small_nn * 8 + 16;
      // path sums in the reference's order: Floyd-Warshall (adjacency input) or Dijkstra (edge dictionaries)
      const bool dj = flags & GK_SP_DIJKSTRA_ORDER;
      GK_CUDA(cudaFuncSetAttribute(spattr_apsp<double>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max<size_t>(smem_a, 16)));
      GK_CUDA(cudaFuncSetAttribute(sp_dijkstra_order_apsp, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max<size_t>(smem_a, 16)));
      if (!small.empty()) {
        pa.glist = lists.as<int>();
        pa.dist_in_global = 0;
        if (dj) sp_dijkstra_order_apsp<<<(int)small.size(), SP_THREADS, smem_a, h->stream>>>(pa);
        else spattr_apsp<double><<<(int)small.size(), SP_THREADS, smem_a, h->stream>>>(pa);
        LAUNCH_CHECK(h);
      }
      if (!big.empty()) {
        pa.glist = lists.as<int>() + small.size();
        pa.dist_in_global = 1;
        if (dj) sp_dijkstra_order_apsp<<<(int)big.size(), SP_THREADS, 16, h->stream>>>(pa);
        else spattr_apsp<double><<<(int)big.size(), SP_THREADS, 16, h->stream>>>(pa);
        LAUNCH_CHECK(h);
      }
      SpParams pb = p;
      pb.gdist = h->sp_dist.p;
      pb.goff = d_goff_all;
      sp_hist_from_dist<<<(int)N, SP_THREADS, SP_LOCAL_SLOTS * 12, h->stream>>>(pb, h->sp_dkeys.as<unsigned long long>(),
                                                                              (unsigned)(dkey_cap - 1));
      LAUNCH_CHECK(h);
    } else {
    if (!small.empty()) {
      p.glist = lists.as<int>();
      p.n_list = (int)small.size();
      p.dist_in_global = 0;
      p.goff = d_goff_all;  // only used for `keep`
      if (use_u16) sp_apsp_hist<unsigned short><<<(int)small.size(), SP_THREADS, smem_small, h->stream>>>(p);
      else sp_apsp_hist<double><<<(int)small.size(), SP_THREADS, smem_small, h->stream>>>(p);
      LAUNCH_CHECK(h);
    }
    // the (up to four) word-width classes are independent: odd classes run on the side stream so
    // that the tail of one launch overlaps the next (they only share atomically updated tables)
    bool forked = false;
    for (int i = 0; i < 4; ++i) {
      if (bfs[i].empty()) continue;
      const int W = 1 << i;
      cudaStream_t st = h->stream;
      if (i & 1) {
        if (!forked) {
          GK_CUDA(cudaEventRecord(h->ev_fork, h->stream));
          GK_CUDA(cudaStreamWaitEvent(h->stream2, h->ev_fork, 0));
          forked = true;
        }
        st = h->stream2;
      }
      int nmax = 0;
      for (int g : bfs[i]) nmax = std::max(nmax, h->graph_ptr_host[g + 1] - h->graph_ptr_host[g]);
      const bool direct = p.n_labels <= SP_DIRECT_MAX_LABELS;
      const size_t smem = (direct ? SP_LOCAL_SLOTS * 4 : SP_LOCAL_SLOTS * 12) + (size_t)nmax * W * 8 + (size_t)16 * W * 8 +
                          (size_t)nmax * 4 + 16;
      p.glist = lists.as<int>() + bfs_off[i];
      p.n_list = (int)bfs[i].size();
      p.dist_in_global = 0;
      p.goff = d_goff_all;
      const int threads = nmax <= 32 ? 32 : nmax <= 64 ? 64 : 128;
      switch (W) {
        case 1: GK_CUDA(cudaFuncSetAttribute(sp_bfs_hist<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); break;
        case 2: GK_CUDA(cudaFuncSetAttribute(sp_bfs_hist<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); break;
        case 4: GK_CUDA(cudaFuncSetAttribute(sp_bfs_hist<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); break;
        default: GK_CUDA(cudaFuncSetAttribute(sp_bfs_hist<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); break;
      }
      switch (W) {
        case 1: sp_bfs_hist<1><<<(int)bfs[i].size(), threads, smem, st>>>(p); break;
        case 2: sp_bfs_hist<2><<<(int)bfs[i].size(), threads, smem, st>>>(p); break;
        case 4: sp_bfs_hist<4><<<(int)bfs[i].size(), threads, smem, st>>>(p); break;
        default: sp_bfs_hist<8><<<(int)bfs[i].size(), threads, smem, st>>>(p); break;
      }
      LAUNCH_CHECK(h);
    }
    if (forked) {
      GK_CUDA(cudaEventRecord(h->ev_join, h->stream2));
      GK_CUDA(cudaStreamWaitEvent(h->stream, h->ev_join, 0));
    }
    if (!big.empty()) {
      if (keep) return fail(GK_ERR_UNSUPPORTED, "gk_sp_features: KEEP_DIST with graphs beyond the shared-memory budget");
      p.glist = lists.as<int>() + small.size();
      p.n_list = (int)big.size();
      p.dist_in_global = 1;
      p.goff = d_goff_big;
      if (use_u16) sp_apsp_hist<unsigned short><<<(int)big.size(), SP_THREADS, smem_big, h->stream>>>(p);
      else sp_apsp_hist<double><<<(int)big.size(), SP_THREADS, smem_big, h->stream>>>(p);
      LAUNCH_CHECK(h);
    }
    }  // integer-distance mode
    }  // passes (WL levels)
    DevScalars* hs;
    GK_TRY(read_scalars(h, &hs));
    if (hs->sp_nonint && !real_mode) { real_mode = true; --attempt; continue; }  // switch to exact float keys
    if (hs->ft_overflow & 8u) {  // real mode: the distance dictionary is full (features of this attempt incomplete)
      if (dkey_cap >= DKEY_CAP_MAX)
        return fail(GK_ERR_UNSUPPORTED, "gk_sp_features: more than 2^24 distinct real-valued path lengths");
      dkey_cap = std::min(dkey_cap * 8, DKEY_CAP_MAX);
      if (hs->ft_overflow & 2u) dict_cap *= 8;
      continue;
    }
    if (hs->ft_overflow & 2u) { dict_cap *= 8; continue; }
    if (hs->ft_overflow & 1u) { ft_cap *= 4; continue; }
    if ((size_t)hs->sp_dict_size * 2 > dict_cap) { dict_cap *= 4; continue; }  // keep probe chains short
    break;
  }
  GK_CUDA(cudaEventRecord(h->tev[3], h->stream));
  GK_CUDA(cudaEventSynchronize(h->tev[3]));
  DevScalars* hs = h->h_scalars.as<DevScalars>();
  h->n_columns = (int64_t)dict_cap;  // column id = dictionary slot
  features_publish(h, FK_SP);
  if (stats) {
    memset(stats, 0, sizeof(*stats));
    stats->n_graphs = h->N; stats->n_vertices = h->V; stats->n_edges = h->E;
    stats->n_levels = 1;
    stats->level_dims[0] = hs->sp_dict_size;
    stats->n_columns = hs->sp_dict_size;
    stats->kernel_launches = h->launches - launches0;
    stats->ms_features = ev_ms(h->tev[2], h->tev[3]);
  }
  return GK_OK;
}

int gk_sp_features(gk_handle* h, int32_t flags, gk_stats* stats) {
  GK_TRY(sp_check(h, flags));
  return sp_features_impl(h, flags, SpLabels(), stats);
}

int gk_wl_sp_features(gk_handle* h, int32_t n_iter, int32_t flags, gk_stats* stats) {
  if (n_iter < 0) return fail(GK_ERR_ARG, "gk_wl_sp_features: n_iter out of range");
  flags |= GK_SP_WITH_LABELS;
  GK_TRY(sp_check(h, flags));
  gk_stats wst;
  GK_TRY(gk_wl_features(h, n_iter, &wst));
  features_begin(h);
  if (h->wl_sparse_ids) {  // the base kernel's counters are indexed by dense label ids
    for (int lv = 1; lv <= n_iter; ++lv) GK_TRY(wl_densify(h, lv, h->labels_all.as<int>() + (size_t)lv * h->V));
    h->wl_sparse_ids = false;
  }
  SpLabels lab;
  lab.n_pass = n_iter + 1;
  lab.labels = h->labels_all.as<int>();
  lab.level_base.assign(lab.n_pass + 1, 0);
  for (int l = 0; l < lab.n_pass; ++l) lab.level_base[l + 1] = lab.level_base[l] + wst.level_dims[l];
  return sp_features_impl(h, flags, lab, stats);
}

// ---------------------------------------------------------------------------
// HadamardCode (hadamard_code.cuh): the vectors of levels 0 .. upto into the two halves of hc_S (level i in half i & 1).
// With `fst`, every level's classes are resolved into dense ids in labels_all, and with `count` also counted into the
// per-level sub-tables of the feature block.
static int hc_run_levels(gk_handle* h, int upto, const FeatStats* fst, bool count, size_t ft_level_cap) {
  const int V = (int)h->V;
  int lgW = 0;
  while ((1 << lgW) < h->hc_W) ++lgW;
  HcShape s;
  s.V = V; s.lgW = lgW; s.lgT = std::min(lgW, 5);
  const int nbT = cdiv((long long)V << s.lgT, HC_THREADS), nb = cdiv(V, 256);
  unsigned long long* S[2] = {h->hc_S.as<unsigned long long>(), h->hc_S.as<unsigned long long>() + ((size_t)V << lgW)};
  const unsigned long long* z = h->hc_z.as<unsigned long long>();
  const unsigned char* skip = h->hc_has_skip ? h->hc_skip.as<unsigned char>() : nullptr;
  unsigned long long* keys = fst ? h->ht_keys.as<unsigned long long>() : nullptr;
  int* rep = h->ht_rep.as<int>();
  const unsigned mask = (unsigned)(h->ht_cap - 1);
  DevScalars* sc = h->scalars.as<DevScalars>();
  for (int lv = 0; lv <= upto; ++lv) {
    if (fst) {
      GK_CUDA(cudaMemsetAsync(h->ht_keys.p, 0xFF, h->ht_cap * 8, h->stream));
      GK_CUDA(cudaMemsetAsync(h->ht_rep.p, 0x7F, h->ht_cap * 4, h->stream));
    }
    if (lv == 0)
      hc_level0<<<nbT, HC_THREADS, 0, h->stream>>>(s, h->labels0.as<int>(), z, S[0], keys, rep, mask, h->slot_of.as<int>(), sc);
    else
      hc_step<<<nbT, HC_THREADS, 0, h->stream>>>(s, h->row_ptr.as<int>(), h->col_idx.as<int>(), skip, z, S[(lv - 1) & 1],
                                                  S[lv & 1], keys, rep, mask, h->slot_of.as<int>(), sc);
    LAUNCH_CHECK(h);
    if (!fst) continue;
    const unsigned char* lv_skip = lv ? skip : nullptr;  // level 0 holds every labelled vertex
    hc_verify<<<nbT, HC_THREADS, 0, h->stream>>>(s, lv_skip, S[lv & 1], rep, h->slot_of.as<int>(), h->flags.as<int>(), sc);
    LAUNCH_CHECK(h);
    hc_flag_sums<<<nb, 256, 0, h->stream>>>(V, h->flags.as<int>(), h->block_sums.as<int>());
    LAUNCH_CHECK(h);
    int* lab_out = h->labels_all.as<int>() + (size_t)lv * V;
    wl_assign<<<nb, 256, 0, h->stream>>>(V, lv, h->flags.as<int>(), h->block_sums.as<int>(), lab_out, sc);
    LAUNCH_CHECK(h);
    hc_gather_insert<<<nb, 256, 0, h->stream>>>(V, lv, lv_skip, h->slot_of.as<int>(), lab_out, h->vgraph.as<int>(), *fst,
                                                count ? h->ft_keys.as<unsigned long long>() : nullptr,
                                                h->ft_cnt.as<unsigned>(), (unsigned)(ft_level_cap - 1));
    LAUNCH_CHECK(h);
  }
  return GK_OK;
}

int gk_hc_features(gk_handle* h, int32_t n_iter, int32_t width, const uint8_t* skip, int32_t flags, gk_stats* stats) {
  GK_TRY(need_packed(h, "gk_hc_features"));
  if (!h->has_labels || h->V == 0) return fail(GK_ERR_ARG, "gk_hc_features: vertex labels are required");
  if (n_iter < 1 || n_iter >= MAX_LEVELS) return fail(GK_ERR_ARG, "gk_hc_features: n_iter out of range [1, 64)");
  if (width < 1 || (width & (width - 1))) return fail(GK_ERR_ARG, "gk_hc_features: width must be a power of two");
  if (h->n_labels0 > width) return fail(GK_ERR_ARG, "gk_hc_features: a packed label is >= width");
  if (flags & ~(GK_HC_SP | GK_SP_DIJKSTRA_ORDER)) return fail(GK_ERR_ARG, "gk_hc_features: unknown flags");
  const bool sp = flags & GK_HC_SP;
  const int64_t V = h->V;
  if (sp && skip)
    for (int64_t v = 0; v < V; ++v)
      if (skip[v]) return fail(GK_ERR_ARG, "gk_hc_features: the ShortestPath base needs a label for every vertex at every level");
  const double need = 2.0 * (double)V * (double)width * 8.0;
  {
    size_t free_b = 0, total_b = 0;
    GK_CUDA(cudaMemGetInfo(&free_b, &total_b));
    if (need > (double)free_b + (double)h->hc_S.cap)
      return fail(GK_ERR_UNSUPPORTED, "gk_hc_features: the two level buffers of V x W x 8 bytes need " +
                                          std::to_string((long long)(need / 1048576.0)) + " MiB, " +
                                          std::to_string((long long)((free_b + h->hc_S.cap) / 1048576)) + " MiB are available");
  }
  const int L = n_iter;
  const int nb = cdiv(V, 256);
  const int64_t launches0 = h->launches;
  features_begin(h);
  h->hc_W = 0;
  GK_TRY(h->hc_S.ensure((size_t)need));
  GK_TRY(h->hc_z.ensure((size_t)width * 8));
  h->hc_has_skip = skip != nullptr;
  if (skip) {
    GK_TRY(h->hc_skip.ensure((size_t)V));
    GK_CUDA(cudaMemcpyAsync(h->hc_skip.p, skip, (size_t)V, cudaMemcpyHostToDevice, h->stream));
  }
  GK_TRY(h->labels_all.ensure((size_t)L * V * 4));
  GK_TRY(h->slot_of.ensure(V * 4));
  GK_TRY(h->flags.ensure(V * 4));
  GK_TRY(h->block_sums.ensure((size_t)nb * 4));
  h->ht_cap = std::max<size_t>(next_pow2((size_t)V * 2), 1024);
  GK_TRY(h->ht_keys.ensure(h->ht_cap * 8));
  GK_TRY(h->ht_rep.ensure(h->ht_cap * 4));
  const size_t ft_level_cap = std::max<size_t>(next_pow2((size_t)V * 2), 1024);
  if (!sp) {
    if (ft_level_cap * (size_t)L > (1ULL << 31)) return fail(GK_ERR_ARG, "gk_hc_features: feature table too large");
    h->ft_cap = ft_level_cap * (size_t)L;
    GK_TRY(h->ft_keys.ensure(h->ft_cap * 8));
    GK_TRY(h->ft_cnt.ensure(h->ft_cap * 4));
  }
  h->hc_W = width;
  h->hc_levels = L;
  std::vector<unsigned long long> z((size_t)width);
  int retries = 0;
  GK_CUDA(cudaEventRecord(h->tev[2], h->stream));
  for (;; ++retries) {
    if (retries > 8) return fail(GK_ERR_STATE, "gk_hc_features: repeated hash collisions");
    const unsigned long long seed = mix64(0x2545F4914F6CDD1DULL + 0x9E3779B97F4A7C15ULL * (unsigned long long)retries);
    const bool degenerate = retries == 0 && h->hc_degenerate_once;
    for (int c = 0; c < width; ++c) z[c] = degenerate ? 0ULL : (mix64(seed + 0xD1B54A32D192ED03ULL * (unsigned long long)(c + 1)) | 1ULL);
    GK_CUDA(cudaMemcpyAsync(h->hc_z.p, z.data(), (size_t)width * 8, cudaMemcpyHostToDevice, h->stream));
    GK_TRY(init_scalars(h, 0));  // (synchronises: z may be rewritten by the next attempt)
    FeatStats fst;
    GK_TRY(reset_feature_stats(h, V * (int64_t)L + 1, (int64_t)nb * L, &fst));
    if (!sp) {
      GK_CUDA(cudaMemsetAsync(h->ft_keys.p, 0xFF, h->ft_cap * 8, h->stream));
      GK_CUDA(cudaMemsetAsync(h->ft_cnt.p, 0, h->ft_cap * 4, h->stream));
    }
    GK_TRY(hc_run_levels(h, L - 1, &fst, !sp, ft_level_cap));
    DevScalars* hs;
    GK_TRY(read_scalars(h, &hs));
    if (hs->ft_overflow) return fail(GK_ERR_STATE, "gk_hc_features: hash table overflow");
    if (!hs->collision) break;
  }
  h->hc_degenerate_once = false;
  GK_CUDA(cudaEventRecord(h->tev[3], h->stream));
  GK_CUDA(cudaEventSynchronize(h->tev[3]));
  const float ms_relabel = ev_ms(h->tev[2], h->tev[3]);
  const DevScalars hs = *h->h_scalars.as<DevScalars>();
  h->n_levels = L;
  h->wl_sparse_ids = false;
  if (sp) {
    SpLabels lab;
    lab.n_pass = L;
    lab.labels = h->labels_all.as<int>();
    lab.level_base.assign(hs.level_base, hs.level_base + L + 1);
    GK_TRY(sp_features_impl(h, GK_SP_WITH_LABELS | (flags & GK_SP_DIJKSTRA_ORDER), lab, stats));
    if (stats) {
      stats->hash_retries = retries;
      stats->ms_hash = ms_relabel;
      stats->kernel_launches = h->launches - launches0;
    }
    return GK_OK;
  }
  h->n_columns = hs.level_base[L];
  features_publish(h, FK_WL);
  if (stats) {
    memset(stats, 0, sizeof(*stats));
    stats->n_graphs = h->N; stats->n_vertices = V; stats->n_edges = h->E;
    stats->n_levels = L;
    for (int i = 0; i < L; ++i) stats->level_dims[i] = hs.level_dims[i];
    stats->n_columns = h->n_columns;
    stats->hash_retries = retries;
    stats->kernel_launches = h->launches - launches0;
    stats->ms_features = ms_relabel;
    stats->ms_hash = ms_relabel;
  }
  return GK_OK;
}

int gk_hc_vectors(gk_handle* h, int32_t level, int64_t* out) {
  if (!h || !out) return fail(GK_ERR_ARG, "gk_hc_vectors: null argument");
  if (h->hc_W <= 0 || level < 0 || level >= h->hc_levels)
    return fail(GK_ERR_STATE, "gk_hc_vectors: no such level (run gk_hc_features on the packed block first)");
  GK_CUDA(cudaSetDevice(h->dev));
  GK_TRY(hc_run_levels(h, level, nullptr, false, 0));
  const size_t n = (size_t)h->V * (size_t)h->hc_W;
  GK_CUDA(cudaMemcpyAsync(out, h->hc_S.as<unsigned long long>() + (size_t)(level & 1) * n, n * 8, cudaMemcpyDeviceToHost,
                          h->stream));
  GK_CUDA(cudaStreamSynchronize(h->stream));
  return GK_OK;
}

int gk_selftest_hc_collision(gk_handle* h) {
  if (!h) return fail(GK_ERR_ARG, "null handle");
  h->hc_degenerate_once = true;
  return GK_OK;
}

int gk_selftest_wl_collision(gk_handle* h, int32_t attempts, int32_t from_level) {
  if (!h) return fail(GK_ERR_ARG, "null handle");
  if (attempts < 0 || from_level < 1) return fail(GK_ERR_ARG, "gk_selftest_wl_collision: bad arguments");
  h->wl_degen_attempts = attempts;
  h->wl_degen_from = from_level;
  return GK_OK;
}

int gk_sp_distances(gk_handle* h, int64_t g, double* out) {
  if (!h || !out) return fail(GK_ERR_ARG, "gk_sp_distances: null argument");
  if (h->feature_kind == FK_SPATTR && h->sp_dist_esz) {
    // after gk_spattr_features: the APSP matrices of every graph are still in sp_dist (u16 with the saturated
    // value 0x3FFF for "no path", or fp64 with +inf)
    if (g < 0 || g >= h->N) return fail(GK_ERR_ARG, "gk_sp_distances: bad graph index");
    const long long off = h->sp_goff[g], cnt = h->sp_goff[g + 1] - off;
    GK_CUDA(cudaSetDevice(h->dev));
    if (h->sp_dist_esz == 8) {
      GK_CUDA(cudaMemcpyAsync(out, h->sp_dist.as<double>() + off, cnt * 8, cudaMemcpyDeviceToHost, h->stream));
      GK_CUDA(cudaStreamSynchronize(h->stream));
    } else {
      std::vector<unsigned short> tmp((size_t)cnt);
      GK_CUDA(cudaMemcpyAsync(tmp.data(), h->sp_dist.as<unsigned short>() + off, cnt * 2, cudaMemcpyDeviceToHost, h->stream));
      GK_CUDA(cudaStreamSynchronize(h->stream));
      for (long long i = 0; i < cnt; ++i) out[i] = tmp[i] < 0x3FFF ? (double)tmp[i] : INFINITY;
    }
    return GK_OK;
  }
  if (h->feature_kind != FK_SP || !(h->sp_flags & GK_SP_KEEP_DIST)) return fail(GK_ERR_STATE, "gk_sp_distances: run gk_sp_features with GK_SP_KEEP_DIST (or gk_spattr_features) first");
  if (g < 0 || g >= h->N) return fail(GK_ERR_ARG, "gk_sp_distances: bad graph index");
  const long long off = h->sp_goff[g], cnt = h->sp_goff[g + 1] - off;
  GK_CUDA(cudaSetDevice(h->dev));
  GK_CUDA(cudaMemcpyAsync(out, h->K_stage.as<double>() + off, cnt * 8, cudaMemcpyDeviceToHost, h->stream));
  GK_CUDA(cudaStreamSynchronize(h->stream));
  return GK_OK;
}

int gk_spattr_features(gk_handle* h, int32_t flags, gk_stats* stats) {
  GK_TRY(need_packed(h, "gk_spattr_features"));
  if (!h->attrs.p || h->attr_dim <= 0) return fail(GK_ERR_ARG, "gk_spattr_features: node attributes are required");
  const int64_t N = h->N;
  const int da = h->attr_dim, dd = da * da;
  if (dd > 1024) return fail(GK_ERR_UNSUPPORTED, "gk_spattr_features: attribute dimension above 32");
  const bool use_u16 = (!h->has_weights || h->unit_weights) && h->max_graph_size < 16000;
  const size_t esz = use_u16 ? 2 : 8;
  const int64_t launches0 = h->launches;
  features_begin(h);
  if ((size_t)h->max_graph_size * h->max_graph_size * 2 + (size_t)h->max_graph_size * da * 8 + (size_t)dd * 8 > 200 * 1024)
    return fail(GK_ERR_UNSUPPORTED, "gk_spattr_features: graph too large for the shared-memory feature kernel");

  // per-graph offsets of the distance matrices (all kept in global memory for phase C)
  std::vector<int> small, big;
  size_t max_small_nn = 0;
  h->sp_goff.assign(N + 1, 0);
  long long off_all = 0;
  for (int64_t g = 0; g < N; ++g) {
    const long long n = h->graph_ptr_host[g + 1] - h->graph_ptr_host[g];
    h->sp_goff[g] = off_all;
    off_all += n * n;
    if ((size_t)(n * n) * esz <= 160 * 1024) { small.push_back((int)g); max_small_nn = std::max(max_small_nn, (size_t)(n * n)); }
    else big.push_back((int)g);
  }
  h->sp_goff[N] = off_all;
  std::vector<int> order(small);
  order.insert(order.end(), big.begin(), big.end());
  GK_TRY(h->sp_lists.ensure((size_t)N * 4 + 16));
  GK_CUDA(cudaMemcpyAsync(h->sp_lists.p, order.data(), order.size() * 4, cudaMemcpyHostToDevice, h->stream));
  GK_TRY(h->sp_graph_off.ensure((size_t)(N + 1) * 8));
  GK_CUDA(cudaMemcpyAsync(h->sp_graph_off.p, h->sp_goff.data(), (N + 1) * 8, cudaMemcpyHostToDevice, h->stream));
  GK_TRY(h->sp_dist.ensure((size_t)std::max<long long>(off_all, 1) * esz));
  const size_t dict_cap = 1 << 16;
  GK_TRY(h->sp_dict_keys.ensure(dict_cap * 8));
  GK_TRY(h->sp_dict_ids.ensure(dict_cap * 4));
  h->sp_dict_cap = dict_cap;
  GK_TRY(init_scalars(h, 0));
  GK_CUDA(cudaMemsetAsync(h->sp_dict_keys.p, 0xFF, dict_cap * 8, h->stream));
  GK_CUDA(cudaStreamSynchronize(h->stream));

  GK_CUDA(cudaEventRecord(h->tev[2], h->stream));
  SpParams p;
  memset(&p, 0, sizeof(p));
  p.graph_ptr = h->graph_ptr.as<int>();
  p.row_ptr = h->row_ptr.as<int>();
  p.col_idx = h->col_idx.as<int>();
  p.weights = (h->has_weights && !use_u16) ? h->weights.as<double>() : nullptr;
  p.gdist = h->sp_dist.p;
  p.goff = h->sp_graph_off.as<long long>();
  p.dict_keys = h->sp_dict_keys.as<unsigned long long>();
  p.dict_mask = (unsigned)(dict_cap - 1);
  p.sc = h->scalars.as<DevScalars>();
  const size_t smem_small = max_small_nn * esz + 16;
  const bool dj = !use_u16 && (flags & GK_SP_DIJKSTRA_ORDER);  // real-valued weights: path sums in Dijkstra's order
  if (use_u16) GK_CUDA(cudaFuncSetAttribute(spattr_apsp<unsigned short>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_small));
  else if (dj) GK_CUDA(cudaFuncSetAttribute(sp_dijkstra_order_apsp, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_small));
  else GK_CUDA(cudaFuncSetAttribute(spattr_apsp<double>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_small));
  if (!small.empty()) {
    p.glist = h->sp_lists.as<int>();
    p.dist_in_global = 0;
    if (use_u16) spattr_apsp<unsigned short><<<(int)small.size(), SP_THREADS, smem_small, h->stream>>>(p);
    else if (dj) sp_dijkstra_order_apsp<<<(int)small.size(), SP_THREADS, smem_small, h->stream>>>(p);
    else spattr_apsp<double><<<(int)small.size(), SP_THREADS, smem_small, h->stream>>>(p);
    LAUNCH_CHECK(h);
  }
  if (!big.empty()) {
    p.glist = h->sp_lists.as<int>() + small.size();
    p.dist_in_global = 1;
    if (use_u16) spattr_apsp<unsigned short><<<(int)big.size(), SP_THREADS, 16, h->stream>>>(p);
    else if (dj) sp_dijkstra_order_apsp<<<(int)big.size(), SP_THREADS, 16, h->stream>>>(p);
    else spattr_apsp<double><<<(int)big.size(), SP_THREADS, 16, h->stream>>>(p);
    LAUNCH_CHECK(h);
  }
  // distinct distances -> block ids (ascending distance order, deterministic)
  std::vector<unsigned long long> keys(dict_cap);
  GK_CUDA(cudaMemcpyAsync(keys.data(), h->sp_dict_keys.p, dict_cap * 8, cudaMemcpyDeviceToHost, h->stream));
  DevScalars* hs;
  GK_TRY(read_scalars(h, &hs));
  // block ids are 16-bit in spattr_accumulate; a full 65536-slot dictionary is past that limit as well
  if (hs->ft_overflow || hs->sp_dkey_size > 32768)
    return fail(GK_ERR_UNSUPPORTED, "gk_spattr_features: more than 32768 distinct path lengths");
  std::vector<std::pair<double, int>> found;
  for (size_t i = 0; i < dict_cap; ++i)
    if (keys[i] != EMPTY64) {
      double d;
      if (use_u16) d = (double)keys[i];
      else { long long b = (long long)keys[i]; memcpy(&d, &b, 8); }
      found.emplace_back(d, (int)i);
    }
  std::sort(found.begin(), found.end());
  const int n_blocks = (int)found.size();
  std::vector<int> slot_block(dict_cap, -1);
  for (int b = 0; b < n_blocks; ++b) slot_block[found[b].second] = b;
  GK_CUDA(cudaMemcpyAsync(h->sp_dict_ids.p, slot_block.data(), dict_cap * 4, cudaMemcpyHostToDevice, h->stream));
  const int64_t Dfeat = (int64_t)std::max(n_blocks, 1) * dd;
  if ((size_t)N * Dfeat * 8 > (size_t)64 << 30) return fail(GK_ERR_UNSUPPORTED, "gk_spattr_features: feature matrix above 64 GB");
  GK_TRY(h->fattr.ensure((size_t)N * Dfeat * 8));
  GK_CUDA(cudaMemsetAsync(h->fattr.p, 0, (size_t)N * Dfeat * 8, h->stream));
  h->fattr_dim = Dfeat;
  if (n_blocks > 0) {
    const size_t fixed = (size_t)h->max_graph_size * da * 8 + (size_t)h->max_graph_size * h->max_graph_size * 2 + 64;
    int chunk = (int)std::min<size_t>((size_t)n_blocks, (200 * 1024 - fixed) / ((size_t)dd * 8));
    if (chunk < 1) return fail(GK_ERR_UNSUPPORTED, "gk_spattr_features: shared memory budget exceeded");
    const size_t smem = (size_t)chunk * dd * 8 + fixed;
    if (use_u16) {
      GK_CUDA(cudaFuncSetAttribute(spattr_accumulate<unsigned short>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      spattr_accumulate<unsigned short><<<(int)N, 256, smem, h->stream>>>(
          h->graph_ptr.as<int>(), h->attrs.as<double>(), da, h->sp_dist.p, h->sp_graph_off.as<long long>(),
          h->sp_dict_keys.as<unsigned long long>(), (unsigned)(dict_cap - 1), h->sp_dict_ids.as<int>(), n_blocks, chunk,
          h->fattr.as<double>());
    } else {
      GK_CUDA(cudaFuncSetAttribute(spattr_accumulate<double>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      spattr_accumulate<double><<<(int)N, 256, smem, h->stream>>>(
          h->graph_ptr.as<int>(), h->attrs.as<double>(), da, h->sp_dist.p, h->sp_graph_off.as<long long>(),
          h->sp_dict_keys.as<unsigned long long>(), (unsigned)(dict_cap - 1), h->sp_dict_ids.as<int>(), n_blocks, chunk,
          h->fattr.as<double>());
    }
    LAUNCH_CHECK(h);
  }
  GK_TRY(h->diag_f64.ensure(N * 8));
  DevScalars* sc = h->scalars.as<DevScalars>();
  rownorm_f64_kernel<<<(int)N, 256, 0, h->stream>>>(h->fattr.as<double>(), Dfeat, (int)N, h->diag_f64.as<double>(),
                                                     &sc->fattr_negative);
  LAUNCH_CHECK(h);
  GK_CUDA(cudaEventRecord(h->tev[3], h->stream));
  unsigned* h_negative = &h->h_scalars.as<DevScalars>()->fattr_negative;
  GK_CUDA(cudaMemcpyAsync(h_negative, &sc->fattr_negative, sizeof(unsigned), cudaMemcpyDeviceToHost, h->stream));
  GK_CUDA(cudaStreamSynchronize(h->stream));  // host vectors above are sources of async copies
  h->fattr_signed = *h_negative != 0;
  h->n_columns = Dfeat;
  h->sp_dist_esz = (int)esz;
  features_publish(h, FK_SPATTR);
  if (stats) {
    memset(stats, 0, sizeof(*stats));
    stats->n_graphs = N; stats->n_vertices = h->V; stats->n_edges = h->E;
    stats->n_levels = 1;
    stats->level_dims[0] = n_blocks;
    stats->n_columns = Dfeat;
    stats->n_dense_columns = Dfeat;
    stats->kernel_launches = h->launches - launches0;
    stats->ms_features = ev_ms(h->tev[2], h->tev[3]);
  }
  return GK_OK;
}

static void build_tiles(std::vector<int2>& tiles, int a0, int a1, int b0, int b1, bool upper_only, int bm);

// ---------------------------------------------------------------------------
// One gk_gram request, checked by gram_request and handed to the route of the feature kind.
struct GramReq {
  int64_t N;           // rows of the feature block (gk_set_row_map)
  const int* row_map;  // packed graph -> row of the block, null for the identity
  int64_t n_fit, k_rows, k_cols, row_begin, row_end;
  int a0, a1;          // K's rows are the block's rows [a0, a1)
  bool square, full_square, dev_out;
  int64_t ld;          // resolved: >= k_cols
  int32_t flags, out_dtype;
  void* K_out;
  double *xdiag, *ydiag;
};

// What each feature kind's route accepts besides fp64 host output of a row range of K.
struct GramRules {
  const char* name;
  bool f32_out, dev_out, row_map, dist;
};
static const GramRules GRAM_RULES[] = {
    /* FK_NONE   */ {"integer", true, true, true, true},
    /* FK_WL     */ {"WL", true, true, true, true},
    /* FK_SP     */ {"ShortestPath", true, true, true, true},
    /* FK_SPATTR */ {"ShortestPathAttr", false, false, false, false},
    /* FK_GH     */ {"GraphHopper", false, false, false, false},
    /* FK_NH     */ {"NeighborhoodHash", false, true, false, false},
    /* FK_RW     */ {"random walk", false, true, false, false},
    /* FK_PK     */ {"Propagation", true, true, false, false},
    /* FK_PM     */ {"PyramidMatch", false, true, false, false},
    /* FK_NSPD   */ {"NeighborhoodSubgraphPairwiseDistance", false, true, false, false},
    /* FK_SM     */ {"SubgraphMatching", false, true, false, false},
    /* FK_ODD    */ {"OddSth", false, true, false, false},
    /* FK_ML     */ {"MultiscaleLaplacian", false, true, false, false},
    /* FK_SVMT   */ {"SvmTheta", false, true, false, false},
    /* FK_GS     */ {"GraphletSampling", false, true, false, false},
};

static int gram_request(gk_handle* h, FeatureKind kind, int64_t n_fit, int32_t flags, int64_t row_begin,
                        int64_t row_end, void* K_out, int32_t out_dtype, int64_t ld, double* xdiag, double* ydiag,
                        GramReq* q) {
  const GramRules& r = GRAM_RULES[kind];
  if (out_dtype != GK_F32 && out_dtype != GK_F64) return fail(GK_ERR_ARG, "gk_gram: bad out_dtype");
  // MultiscaleLaplacian's and SvmTheta's rows are their records: the fitted graphs' (kept from the fit), then the new ones
  const int64_t N = h->n_rows > 0 ? h->n_rows : kind == FK_ML ? h->ml_nrec : kind == FK_SVMT ? h->svmt_nrec : h->N;
  if (n_fit <= 0 || n_fit > N) return fail(GK_ERR_ARG, "gk_gram: n_fit out of range");
  const bool dist = (flags & (GK_DIST | GK_DIST_GATHER)) != 0;
  if (h->n_rows > 0 && !r.row_map) return fail(GK_ERR_UNSUPPORTED, std::string("gk_gram: row map with ") + r.name + " features");
  if (dist && !r.dist) return fail(GK_ERR_UNSUPPORTED, std::string("gk_gram: GK_DIST with ") + r.name + " features");
  if (out_dtype != GK_F64 && !r.f32_out) return fail(GK_ERR_UNSUPPORTED, std::string(r.name) + " Gram is fp64 only");
  if ((flags & GK_OUT_DEVICE) && !r.dev_out)
    return fail(GK_ERR_UNSUPPORTED, std::string(r.name) + " Gram: device output not supported");
  const bool square = n_fit == N;
  const int64_t k_rows_total = square ? N : N - n_fit;
  if (row_end < 0) row_end = k_rows_total;
  if (row_begin < 0 || row_begin > row_end || row_end > k_rows_total) return fail(GK_ERR_ARG, "gk_gram: bad row range");
  if (ld <= 0) ld = n_fit;
  if (ld < n_fit) return fail(GK_ERR_ARG, "gk_gram: ld smaller than the row length");
  if (dist) {  // multi-GPU row tiling of the integer Gram (collective)
    if (!h->comm) return fail(GK_ERR_STATE, "gk_gram: GK_DIST without gk_comm_init");
    if (!square || h->n_rows > 0) return fail(GK_ERR_UNSUPPORTED, "gk_gram: GK_DIST needs the square fit_transform case without a row map");
    if (flags & GK_OUT_DEVICE) return fail(GK_ERR_UNSUPPORTED, "gk_gram: GK_DIST results are library-owned (gk_result_device / gk_fetch / host K_out)");
    int64_t rb = 0, re = 0;
    GK_TRY(gk_comm_rows(h, N, &rb, &re));
    if (row_begin != rb || row_end != re) return fail(GK_ERR_ARG, "gk_gram: GK_DIST row range must be the one gk_comm_rows returns");
  }
  if ((flags & GK_OUT_DEVICE) && !K_out) return fail(GK_ERR_ARG, "gk_gram: GK_OUT_DEVICE without a pointer");
  q->N = N;
  q->row_map = h->n_rows > 0 ? h->row_map.as<int>() : nullptr;
  q->n_fit = n_fit; q->k_cols = n_fit;
  q->row_begin = row_begin; q->row_end = row_end; q->k_rows = row_end - row_begin;
  q->a0 = (int)((square ? 0 : n_fit) + row_begin); q->a1 = (int)((square ? 0 : n_fit) + row_end);
  q->square = square; q->full_square = square && row_begin == 0 && row_end == N;
  q->dev_out = (flags & GK_OUT_DEVICE) != 0;
  q->ld = ld;
  q->flags = flags; q->out_dtype = out_dtype;
  q->K_out = K_out;
  q->xdiag = xdiag; q->ydiag = ydiag;
  return GK_OK;
}

// The integer feature block gram_int reads: the handle's own (block_of) or one NeighborhoodHash level (gram_nh).
struct IntBlock {
  unsigned long long* keys;  // (graph, column) -> count hash table of `cap` slots
  unsigned* cnt;
  size_t cap;
  unsigned* colcnt;          // graphs per column: col_cap entries, the first n_columns in use
  int64_t col_cap, n_columns;
  unsigned long long* diag;  // self similarities, finished with the n_part per-CTA partials of the feature kernels
  unsigned *part_max, *part_new;
  int64_t n_part;
  bool prologue_on_host;     // gk_wl_features already ran the square Gram prologue of this block
};

static IntBlock block_of(gk_handle* h) {
  IntBlock b;
  b.keys = h->ft_keys.as<unsigned long long>(); b.cnt = h->ft_cnt.as<unsigned>(); b.cap = h->ft_cap;
  b.colcnt = h->colcnt.as<unsigned>(); b.col_cap = h->col_cap; b.n_columns = h->n_columns;
  b.diag = h->diag_u64.as<unsigned long long>();
  b.part_max = h->part_max.as<unsigned>(); b.part_new = h->part_new.as<unsigned>(); b.n_part = h->n_part;
  b.prologue_on_host = h->pro_ready;
  return b;
}

static int gram_int(gk_handle* h, const GramReq& q, const IntBlock& fb, gk_stats* stats);

// Where an fp64 route writes K: the caller's device buffer, else the library-owned h->K with unpitched rows.
struct F64Out {
  double* p;
  int64_t ld;
};

static int f64_target(gk_handle* h, const GramReq& q, F64Out* out) {
  if (q.dev_out) {
    *out = {reinterpret_cast<double*>(q.K_out), q.ld};
    return GK_OK;
  }
  GK_TRY(h->K.ensure((size_t)std::max<int64_t>(q.k_rows, 1) * q.k_cols * 8));
  h->K_rows = q.k_rows; h->K_cols = q.k_cols; h->K_ld = q.k_cols; h->K_dtype = GK_F64;
  *out = {h->K.as<double>(), q.k_cols};
  return GK_OK;
}

// The end of an fp64 route: GK_NORMALIZE by the self similarities in diag_f64 (when the route normalises), ev_d2h,
// the pitched copy of K into the caller's host array, xdiag / ydiag from diag_f64, ev_done (if given), and the
// synchronisation after which the caller's buffers hold the result.
static int f64_deliver(gk_handle* h, const GramReq& q, const F64Out& out, bool normalize, cudaEvent_t ev_d2h,
                       cudaEvent_t ev_done = nullptr) {
  const double* diag = h->diag_f64.as<double>();
  if (normalize && (q.flags & GK_NORMALIZE) && q.k_rows > 0) {
    normalize_rows<double><<<h->sm_count * 8, 256, 0, h->stream>>>(q.k_rows, q.k_cols, out.p, out.ld, diag + q.a0, diag,
                                                                    (q.flags & GK_NAN_TO_NUM) ? 1 : 0);
    LAUNCH_CHECK(h);
  }
  GK_CUDA(cudaEventRecord(ev_d2h, h->stream));
  if (q.K_out && !q.dev_out && q.k_rows > 0)
    GK_CUDA(cudaMemcpy2DAsync(q.K_out, (size_t)q.ld * 8, out.p, (size_t)out.ld * 8, (size_t)q.k_cols * 8,
                              (size_t)q.k_rows, cudaMemcpyDeviceToHost, h->stream));
  if (q.xdiag) GK_CUDA(cudaMemcpyAsync(q.xdiag, diag, q.n_fit * 8, cudaMemcpyDeviceToHost, h->stream));
  if (q.ydiag && !q.square)
    GK_CUDA(cudaMemcpyAsync(q.ydiag, diag + q.n_fit, (q.N - q.n_fit) * 8, cudaMemcpyDeviceToHost, h->stream));
  if (ev_done) GK_CUDA(cudaEventRecord(ev_done, h->stream));
  GK_CUDA(cudaStreamSynchronize(h->stream));
  return GK_OK;
}

// Gram of the dense fp64 SP-attr feature matrix (FK_SPATTR).  Non-negative features: the wgmma kernel with
// tf32 operands on a hi/lo split of the features (3xTF32: hi hi^T + hi lo^T + lo hi^T, fp32 accumulation in
// registers, k range processed in chunks and summed in fp64), self similarities exact in fp64.  Its error is a small
// multiple of 2^-22 times sum_k |phi_ik| |phi_jk| (measured on an H100: below 1e-6 of it), which for non-negative
// features is K_ij itself: every entry within 1e-5 relative.  A feature map with a negative entry (attributes of
// mixed sign) can have entries that cancel far below that scale, so it takes the fp64 CUDA-core Gram (1e-9).
// GRAKEL_B200_SPATTR_F64=1 forces the fp64 Gram, =0 the tensor-core Gram.
static int gram_spattr(gk_handle* h, const GramReq& q, gk_stats* stats) {
  const int64_t N = h->N, n_fit = q.n_fit, k_rows = q.k_rows, k_cols = q.k_cols;
  const bool square = q.square;
  const int a0 = q.a0, a1 = q.a1;
  const int64_t launches0 = h->launches;
  F64Out out;
  GK_TRY(f64_target(h, q, &out));
  GK_CUDA(cudaEventRecord(h->tev[6], h->stream));
  const char* e_f64 = getenv("GRAKEL_B200_SPATTR_F64");
  const bool use_f64 = (e_f64 && *e_f64) ? atoi(e_f64) != 0 : h->fattr_signed;
  if (k_rows > 0 && !use_f64) {
    const long long D = h->fattr_dim, Dp = (D + BK_TF32 - 1) / BK_TF32 * BK_TF32, W = 3 * Dp;
    GK_TRY(h->panel.ensure((size_t)N * W * 4 * 2));
    float* P1 = h->panel.as<float>();
    float* P2 = P1 + (size_t)N * W;
    spattr_split_tf32<<<h->sm_count * 8, 256, 0, h->stream>>>(h->fattr.as<double>(), D, Dp, (int)N, P1, P2);
    LAUNCH_CHECK(h);
    const bool sym = q.full_square;
    std::vector<int2> tiles;
    build_tiles(tiles, a0, a1, 0, (int)n_fit, sym, BM);
    GK_TRY(h->h_tiles.ensure(tiles.size() * sizeof(int2)));
    memcpy(h->h_tiles.p, tiles.data(), tiles.size() * sizeof(int2));
    GK_TRY(h->tiles.ensure(tiles.size() * sizeof(int2)));
    GK_CUDA(cudaMemcpyAsync(h->tiles.p, h->h_tiles.p, tiles.size() * sizeof(int2), cudaMemcpyHostToDevice, h->stream));
    CUtensorMap tmA, tmB, tmC;
    memset(&tmC, 0, sizeof(tmC));
    GK_TRY(make_panel_map_f32(&tmA, P1, W, N, BM));
    GK_TRY(make_panel_map_f32(&tmB, P2, W, N, BN));
    GramParams p;
    memset(&p, 0, sizeof(p));
    p.tiles = h->tiles.as<int2>();
    p.n_tiles = (int)tiles.size();
    p.a_row_end = a1; p.b_row_end = (int)n_fit;
    p.c_row0 = a0; p.c_col0 = 0;
    p.out = out.p; p.ld = out.ld;
    p.mirror = 0;  // the symmetric case mirrors the upper triangle once, after all chunks (mirror_upper_f64)
    p.diag = h->diag_f64.as<double>();
    // The tensor core's fp32 accumulate truncates, so no accumulator sums more than `chunk` k-blocks x 4 MMAs: the
    // kernel folds every chunk of a tile into the fp64 result itself.
    // Only the hi x hi third of the k range needs short chunks: the two cross thirds are 2^-11 of the sum, their
    // accumulated truncation is 2^-11 of the bound and they go through one accumulator.
    int chunk = 8;
    if (const char* e = getenv("GRAKEL_B200_SPATTR_CHUNK")) chunk = std::max(1, atoi(e));
    p.k_block0 = 0;
    p.num_k_blocks = (int)(W / BK_TF32);
    p.k_chunk = chunk;
    p.k_split = (int)(Dp / BK_TF32);
    p.accumulate = 0;
    const int grid = (int)std::min<size_t>(tiles.size(), h->sm_count);
    gram_tc_kernel<double, false, 1><<<grid, GEMM_THREADS, GEMM_SMEM, h->stream>>>(tmA, tmB, tmC, p);
    LAUNCH_CHECK(h);
    if (sym) {
      mirror_upper_f64<<<h->sm_count * 8, 256, 0, h->stream>>>((int)N, out.p, out.ld);
      LAUNCH_CHECK(h);
    }
    if (square) {  // exact self similarities
      set_diag_f64<<<cdiv(k_rows, 256), 256, 0, h->stream>>>(a0, a1, 0, (int)n_fit, h->diag_f64.as<double>(), out.p, out.ld);
      LAUNCH_CHECK(h);
    }
  }
  if (k_rows > 0 && use_f64) {
    dim3 grid(cdiv(k_cols, 64), cdiv(k_rows, 64));
    gram_f64_kernel<<<grid, 256, 0, h->stream>>>(h->fattr.as<double>(), h->fattr_dim, a0, a1, 0, (int)n_fit, out.p, out.ld);
    LAUNCH_CHECK(h);
  }
  GK_TRY(f64_deliver(h, q, out, true, h->tev[7]));
  if (stats) {
    stats->gram_path = use_f64 ? 5 : 4;
    stats->gemm_launches = h->launches - launches0;
    stats->ms_gemm = ev_ms(h->tev[6], h->tev[7]);
  }
  return GK_OK;
}

}  // extern "C"

// ---- GraphHopper (graph_hopper.cuh)
// Launch one gh_dag_kernel pass over every graph: graphs whose working set fits `smem_cap` bytes of shared memory
// run from shared memory, the others from a global workspace.
template <bool MAPS>
static int gh_dag_pass(gk_handle* h, const std::vector<int>& gdiam, double* M, long long T) {
  const int64_t N = h->N;
  const size_t smem_cap = 96 * 1024;
  std::vector<int> small, big;
  std::vector<long long> woff(N, 0);
  size_t smem_max = 16, ws_total = 0;
  for (int64_t g = 0; g < N; ++g) {
    const long long n = h->graph_ptr_host[g + 1] - h->graph_ptr_host[g];
    const size_t b = gh_ws_bytes(n, MAPS ? gdiam[g] + 1 : 0, MAPS);
    if (b <= smem_cap) { small.push_back((int)g); smem_max = std::max(smem_max, b); }
    else { big.push_back((int)g); woff[g] = (long long)ws_total; ws_total += b; }
  }
  std::vector<int> order(small);
  order.insert(order.end(), big.begin(), big.end());
  GK_TRY(h->sp_lists.ensure((size_t)N * 4 + 16));
  GK_CUDA(cudaMemcpyAsync(h->sp_lists.p, order.data(), order.size() * 4, cudaMemcpyHostToDevice, h->stream));
  GhParams p;
  memset(&p, 0, sizeof(p));
  p.graph_ptr = h->graph_ptr.as<int>();
  p.row_ptr = h->row_ptr.as<int>();
  p.col_idx = h->col_idx.as<int>();
  p.gdiam = h->gh_gdiam.as<int>();
  p.delta_max = h->gh_gdiam.as<int>() + N;
  p.M = M;
  p.delta = h->gh_delta;
  p.T = T;
  if (!big.empty()) {
    GK_TRY(h->gh_ws.ensure(ws_total));
    GK_TRY(h->gh_woff.ensure((size_t)N * 8));
    GK_CUDA(cudaMemcpyAsync(h->gh_woff.p, woff.data(), (size_t)N * 8, cudaMemcpyHostToDevice, h->stream));
  }
  if (!small.empty()) {
    GK_CUDA(cudaFuncSetAttribute(gh_dag_kernel<MAPS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_max));
    p.glist = h->sp_lists.as<int>();
    gh_dag_kernel<MAPS><<<(int)small.size(), GH_THREADS, smem_max, h->stream>>>(p);
    LAUNCH_CHECK(h);
  }
  if (!big.empty()) {
    p.glist = h->sp_lists.as<int>() + small.size();
    p.ws = h->gh_ws.as<unsigned char>();
    p.woff = h->gh_woff.as<long long>();
    p.ws_global = 1;
    gh_dag_kernel<MAPS><<<(int)big.size(), GH_THREADS, 0, h->stream>>>(p);
    LAUNCH_CHECK(h);
  }
  // host vectors above are sources of async copies
  GK_CUDA(cudaStreamSynchronize(h->stream));
  return GK_OK;
}

extern "C" {

int gk_gh_features(gk_handle* h, int32_t node_kernel, double mu, int32_t flags, gk_stats* stats) {
  GK_TRY(need_packed(h, "gk_gh_features"));
  if (!h->attrs.p || h->attr_dim <= 0) return fail(GK_ERR_ARG, "gk_gh_features: node attributes are required");
  if (node_kernel != GK_GH_LINEAR && node_kernel != GK_GH_GAUSSIAN && node_kernel != GK_GH_BRIDGE)
    return fail(GK_ERR_ARG, "gk_gh_features: unknown node kernel");
  if (flags != 0) return fail(GK_ERR_ARG, "gk_gh_features: no flags are defined");
  if (h->has_weights && !h->unit_weights)
    return fail(GK_ERR_UNSUPPORTED, "GraphHopper: edge weights other than 1 (the shortest-path DAG is defined for "
                                    "unweighted graphs only)");
  const int64_t N = h->N, V = h->V;
  const int d = h->attr_dim;
  const int64_t launches0 = h->launches;
  features_begin(h);
  GK_CUDA(cudaEventRecord(h->tev[2], h->stream));
  // pass 1: eccentricities -> per-graph diameter and delta = max diameter + 1
  GK_TRY(h->gh_gdiam.ensure((size_t)(N + 1) * 4));
  GK_CUDA(cudaMemsetAsync(h->gh_gdiam.p, 0, (size_t)(N + 1) * 4, h->stream));
  std::vector<int> gdiam(N + 1, 0);
  GK_TRY(gh_dag_pass<false>(h, gdiam, nullptr, 0));
  GK_CUDA(cudaMemcpyAsync(gdiam.data(), h->gh_gdiam.p, (size_t)(N + 1) * 4, cudaMemcpyDeviceToHost, h->stream));
  GK_CUDA(cudaStreamSynchronize(h->stream));
  const int delta = std::max(gdiam[N], 1);
  const long long T = (long long)delta * (delta + 1) / 2;
  if ((size_t)V * T * 8 > (size_t)64 << 30) return fail(GK_ERR_UNSUPPORTED, "gk_gh_features: node maps above 64 GB");
  h->gh_delta = delta;
  GK_TRY(h->gh_M.ensure((size_t)std::max<int64_t>(V, 1) * T * 8));
  GK_CUDA(cudaMemsetAsync(h->gh_M.p, 0, (size_t)V * T * 8, h->stream));
  // pass 2: the node maps
  GK_TRY(gh_dag_pass<true>(h, gdiam, h->gh_M.as<double>(), T));
  GK_TRY(h->diag_f64.ensure(N * 8));
  int64_t n_columns = T;
  if (node_kernel == GK_GH_LINEAR) {
    // Phi = sum_v vec(M_v) (x) x_v, then the Gram of the SP-attr route (gram_spattr)
    const int64_t D = T * d;
    if ((size_t)N * D * 8 > (size_t)64 << 30) return fail(GK_ERR_UNSUPPORTED, "gk_gh_features: feature matrix above 64 GB");
    GK_TRY(h->fattr.ensure((size_t)N * D * 8));
    gh_linear_features<<<(int)N, 256, 0, h->stream>>>(h->graph_ptr.as<int>(), h->gh_M.as<double>(), T,
                                                      h->attrs.as<double>(), d, h->fattr.as<double>());
    LAUNCH_CHECK(h);
    h->fattr_dim = D;
    n_columns = D;
    DevScalars* sc = h->scalars.as<DevScalars>();
    GK_TRY(init_scalars(h, 0));
    rownorm_f64_kernel<<<(int)N, 256, 0, h->stream>>>(h->fattr.as<double>(), D, (int)N, h->diag_f64.as<double>(),
                                                       &sc->fattr_negative);
    LAUNCH_CHECK(h);
    unsigned* h_negative = &h->h_scalars.as<DevScalars>()->fattr_negative;
    GK_CUDA(cudaMemcpyAsync(h_negative, &sc->fattr_negative, sizeof(unsigned), cudaMemcpyDeviceToHost, h->stream));
    GK_CUDA(cudaEventRecord(h->tev[3], h->stream));
    GK_CUDA(cudaStreamSynchronize(h->stream));
    h->fattr_signed = *h_negative != 0;
  } else {
    if (node_kernel == GK_GH_GAUSSIAN)
      gh_nodepair_diag<GH_NK_GAUSSIAN><<<(int)N, 256, 0, h->stream>>>(h->graph_ptr.as<int>(), h->gh_M.as<double>(), T,
                                                                       h->attrs.as<double>(), d, mu, h->diag_f64.as<double>());
    else
      gh_nodepair_diag<GH_NK_BRIDGE><<<(int)N, 256, 0, h->stream>>>(h->graph_ptr.as<int>(), h->gh_M.as<double>(), T,
                                                                     h->attrs.as<double>(), d, mu, h->diag_f64.as<double>());
    LAUNCH_CHECK(h);
    GK_CUDA(cudaEventRecord(h->tev[3], h->stream));
    GK_CUDA(cudaStreamSynchronize(h->stream));
  }
  h->gh_node_kernel = node_kernel;
  h->gh_mu = mu;
  h->n_columns = n_columns;
  features_publish(h, FK_GH);
  if (stats) {
    memset(stats, 0, sizeof(*stats));
    stats->n_graphs = N; stats->n_vertices = V; stats->n_edges = h->E;
    stats->n_levels = 1;
    stats->level_dims[0] = delta;
    stats->n_columns = n_columns;
    stats->n_dense_columns = node_kernel == GK_GH_LINEAR ? n_columns : 0;
    stats->kernel_launches = h->launches - launches0;
    stats->ms_features = ev_ms(h->tev[2], h->tev[3]);
  }
  return GK_OK;
}

int gk_gh_node_maps(gk_handle* h, int64_t g, double* out) {
  if (!h || !out) return fail(GK_ERR_ARG, "gk_gh_node_maps: null argument");
  if (h->feature_kind != FK_GH) return fail(GK_ERR_STATE, "gk_gh_node_maps: run gk_gh_features first");
  if (g < 0 || g >= h->N) return fail(GK_ERR_ARG, "gk_gh_node_maps: bad graph index");
  const int delta = h->gh_delta;
  const long long T = (long long)delta * (delta + 1) / 2;
  const long long v0 = h->graph_ptr_host[g], n = h->graph_ptr_host[g + 1] - v0;
  std::vector<double> tri((size_t)n * T);
  GK_CUDA(cudaSetDevice(h->dev));
  if (n > 0) {
    GK_CUDA(cudaMemcpyAsync(tri.data(), h->gh_M.as<double>() + v0 * T, (size_t)n * T * 8, cudaMemcpyDeviceToHost, h->stream));
    GK_CUDA(cudaStreamSynchronize(h->stream));
  }
  for (long long v = 0; v < n; ++v) {
    double* o = out + v * delta * delta;
    const double* r = tri.data() + v * T;
    long long k = 0;
    for (int a = 0; a < delta; ++a)
      for (int b = 0; b < delta; ++b) o[a * delta + b] = b >= a ? r[k++] : 0.0;
  }
  return GK_OK;
}

// Consecutive graphs of [g0, g1) in groups of at most GH_GROUP_NODES vertices and GH_GROUP_GRAPHS graphs (a larger
// graph is a group alone).  Appends the first graph of every group and the end.
static void gh_groups(const std::vector<int>& gp, int g0, int g1, std::vector<int>& out) {
  int g = g0;
  while (g < g1) {
    out.push_back(g);
    int e = g + 1;
    while (e < g1 && e - g < GH_GROUP_GRAPHS && gp[e + 1] - gp[g] <= GH_GROUP_NODES) ++e;
    g = e;
  }
  out.push_back(g1);
}

// Gram of the node-pair kernels (gaussian / bridge): gh_nodepair_gram over graph-group pairs, self similarities from
// gh_nodepair_diag.  fp64, host output, GK_NORMALIZE, n_fit / row ranges as in gram_spattr.
static int gram_gh_nodepair(gk_handle* h, const GramReq& q, gk_stats* stats) {
  const int64_t N = h->N, n_fit = q.n_fit, k_rows = q.k_rows;
  const bool square = q.square;
  const int a0 = q.a0, a1 = q.a1;
  const int64_t launches0 = h->launches;
  F64Out out;
  GK_TRY(f64_target(h, q, &out));
  // groups: over all graphs (square) or over Y rows and X columns; the same groups whatever the row range, so a
  // row block reproduces the full matrix's entries bit for bit
  std::vector<int> rgroups, cgroups;
  gh_groups(h->graph_ptr_host, square ? 0 : (int)n_fit, (int)N, rgroups);
  gh_groups(h->graph_ptr_host, 0, (int)n_fit, cgroups);
  const int nrg = (int)rgroups.size() - 1, ncg = (int)cgroups.size() - 1;
  auto touches = [&](int I) { return rgroups[I] < a1 && rgroups[I + 1] > a0; };
  std::vector<int2> pairs;
  for (int I = 0; I < nrg; ++I)
    for (int J = square ? I : 0; J < ncg; ++J)
      if (touches(I) || (square && touches(J))) pairs.push_back(make_int2(I, J));
  GK_CUDA(cudaEventRecord(h->tev[6], h->stream));
  if (k_rows > 0) {
    GK_TRY(h->gh_groups.ensure((rgroups.size() + cgroups.size()) * 4));
    GK_TRY(h->gh_pairs.ensure(std::max<size_t>(pairs.size(), 1) * sizeof(int2)));
    GK_CUDA(cudaMemcpyAsync(h->gh_groups.p, rgroups.data(), rgroups.size() * 4, cudaMemcpyHostToDevice, h->stream));
    GK_CUDA(cudaMemcpyAsync(h->gh_groups.as<int>() + rgroups.size(), cgroups.data(), cgroups.size() * 4,
                            cudaMemcpyHostToDevice, h->stream));
    if (!pairs.empty())
      GK_CUDA(cudaMemcpyAsync(h->gh_pairs.p, pairs.data(), pairs.size() * sizeof(int2), cudaMemcpyHostToDevice, h->stream));
    GhGramParams p;
    memset(&p, 0, sizeof(p));
    p.graph_ptr = h->graph_ptr.as<int>();
    p.M = h->gh_M.as<double>();
    p.T = (long long)h->gh_delta * (h->gh_delta + 1) / 2;
    p.attrs = h->attrs.as<double>();
    p.d = h->attr_dim;
    p.mu = h->gh_mu;
    p.pairs = h->gh_pairs.as<int2>();
    p.rgroups = h->gh_groups.as<int>();
    p.cgroups = h->gh_groups.as<int>() + rgroups.size();
    p.square = square ? 1 : 0;
    p.a0 = a0; p.a1 = a1; p.row0 = a0;
    p.out = out.p;
    p.ld = out.ld;
    if (!pairs.empty()) {
      if (h->gh_node_kernel == GK_GH_GAUSSIAN) {
        GK_CUDA(cudaFuncSetAttribute(gh_nodepair_gram<GH_NK_GAUSSIAN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)GH_GRAM_SMEM));
        gh_nodepair_gram<GH_NK_GAUSSIAN><<<(int)pairs.size(), 256, GH_GRAM_SMEM, h->stream>>>(p);
      } else {
        GK_CUDA(cudaFuncSetAttribute(gh_nodepair_gram<GH_NK_BRIDGE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)GH_GRAM_SMEM));
        gh_nodepair_gram<GH_NK_BRIDGE><<<(int)pairs.size(), 256, GH_GRAM_SMEM, h->stream>>>(p);
      }
      LAUNCH_CHECK(h);
    }
    if (square) {
      set_diag_f64<<<cdiv(k_rows, 256), 256, 0, h->stream>>>(a0, a1, 0, (int)n_fit, h->diag_f64.as<double>(), out.p, out.ld);
      LAUNCH_CHECK(h);
    }
  }
  // its synchronisation also keeps the host group / pair lists alive for their copies
  GK_TRY(f64_deliver(h, q, out, true, h->tev[7]));
  if (stats) {
    stats->gram_path = 6;
    stats->gemm_tiles = (int64_t)pairs.size();
    stats->gemm_launches = h->launches - launches0;
    stats->ms_gemm = ev_ms(h->tev[6], h->tev[7]);
  }
  return GK_OK;
}

// ---------------------------------------------------------------------------
// NeighborhoodHash (neighborhood_hash.cuh).  Level r's expanded block lives at nh_blk + r * nh_level_bytes:
// keys [M] u64 | counts [M] u32 | graphs per column [M + 1] u32 | self similarities [N] u64, M = nh_level_cap (at
// most one unary entry per non-None vertex, so V entries and V columns bound every NeighborhoodHash level;
// PyramidMatch has d entries per vertex).
static size_t nh_level_bytes(int64_t M, int64_t N) {
  const size_t V1 = (size_t)std::max<int64_t>(M, 1);
  const size_t diag_off = (16 * V1 + 4 + 7) / 8 * 8;
  return (diag_off + 8 * (size_t)std::max<int64_t>(N, 1) + 255) / 256 * 256;
}

// Level r's block as an integer feature block; its self similarities are one partial (part_max / part_new, uploaded
// by gram_levels), its column count is set by gram_levels.
static IntBlock nh_level(gk_handle* h, int r) {
  const size_t V1 = (size_t)std::max<int64_t>(h->nh_level_cap, 1);
  char* b = h->nh_blk.as<char>() + (size_t)r * h->nh_level_bytes;
  IntBlock L;
  L.keys = reinterpret_cast<unsigned long long*>(b);
  L.cnt = reinterpret_cast<unsigned*>(b + 8 * V1);
  L.cap = V1;
  L.colcnt = reinterpret_cast<unsigned*>(b + 12 * V1);
  L.col_cap = (int64_t)V1 + 1; L.n_columns = 0;
  L.diag = reinterpret_cast<unsigned long long*>(b + (16 * V1 + 4 + 7) / 8 * 8);
  L.part_max = h->part_max.as<unsigned>(); L.part_new = h->part_new.as<unsigned>(); L.n_part = 1;
  L.prologue_on_host = false;
  return L;
}

// The per-level column pipeline NeighborhoodHash and PyramidMatch share: every level's M entries (codes + valid
// flags) are numbered by distinct code (nh_code_insert / nh_code_number), counted per (graph, column) (nh_count, entry
// e belongs to vertex e / per) and unary-expanded into level block r (oa_colmax / oa_colbase / oa_expand), so that the
// integer Gram of block r gives the levels' multiset intersections.
struct LevelScratch {
  size_t cap, cur_bytes;
  OaCursors* cur;
  unsigned long long* dims;
  int *tab, *colid, *slot_of;
};

static int level_setup(gk_handle* h, int64_t M, int n_blocks, LevelScratch* ls) {
  const int64_t M1 = std::max<int64_t>(M, 1);
  const size_t cap = std::max<size_t>(next_pow2((size_t)M1 * 2), 1024);
  h->nh_level_cap = M1;
  h->nh_level_bytes = nh_level_bytes(M, h->N);
  GK_TRY(h->nh_blk.ensure((size_t)n_blocks * h->nh_level_bytes));
  GK_TRY(h->nh_tab.ensure(cap * 8 + (size_t)M1 * 4));  // slot -> claiming entry | slot -> column | entry -> slot
  GK_TRY(h->ft_keys.ensure(cap * 8));                 // (graph, column) -> count scratch table
  GK_TRY(h->ft_cnt.ensure(cap * 4));
  GK_TRY(h->colmin.ensure((size_t)M1 * 4));  // largest count of every column
  GK_TRY(h->colmax.ensure((size_t)M1 * 4));  // first expanded column of every column
  ls->cap = cap;
  ls->cur_bytes = (size_t)n_blocks * (sizeof(OaCursors) + 8);
  GK_TRY(h->nh_cur.ensure(ls->cur_bytes));
  GK_TRY(h->h_colstats.ensure(std::max(ls->cur_bytes, sizeof(ColStats))));
  ls->cur = h->nh_cur.as<OaCursors>();
  ls->dims = reinterpret_cast<unsigned long long*>(ls->cur + n_blocks);
  ls->tab = h->nh_tab.as<int>();
  ls->colid = ls->tab + cap;
  ls->slot_of = ls->colid + cap;
  GK_CUDA(cudaMemsetAsync(h->nh_cur.p, 0, ls->cur_bytes, h->stream));
  GK_CUDA(cudaMemsetAsync(h->nh_blk.p, 0, (size_t)n_blocks * h->nh_level_bytes, h->stream));
  return GK_OK;
}

static int level_columns(gk_handle* h, const LevelScratch& ls, int r, int64_t M, int per, const unsigned long long* c_r,
                         const unsigned char* v_r) {
  const int64_t M1 = h->nh_level_cap;
  const size_t cap = ls.cap;
  const IntBlock lv = nh_level(h, r);
  GK_CUDA(cudaMemsetAsync(lv.keys, 0xFF, (size_t)M1 * 8, h->stream));
  if (!M) return GK_OK;
  GK_CUDA(cudaMemsetAsync(ls.tab, 0xFF, cap * 4, h->stream));
  GK_CUDA(cudaMemsetAsync(h->ft_keys.p, 0xFF, cap * 8, h->stream));
  GK_CUDA(cudaMemsetAsync(h->ft_cnt.p, 0, cap * 4, h->stream));
  GK_CUDA(cudaMemsetAsync(h->colmin.p, 0, (size_t)M1 * 4, h->stream));
  nh_code_insert<<<cdiv(M, 256), 256, 0, h->stream>>>((int)M, c_r, v_r, ls.tab, (unsigned)(cap - 1), ls.slot_of);
  LAUNCH_CHECK(h);
  nh_code_number<<<cdiv(M, 256), 256, 0, h->stream>>>((int)M, v_r, ls.tab, ls.slot_of, ls.colid, ls.dims + r);
  LAUNCH_CHECK(h);
  nh_count<<<cdiv(M, 256), 256, 0, h->stream>>>((int)M, per, v_r, h->vgraph.as<int>(), ls.slot_of, ls.colid,
                                                h->ft_keys.as<unsigned long long>(), h->ft_cnt.as<unsigned>(),
                                                (unsigned)(cap - 1));
  LAUNCH_CHECK(h);
  oa_colmax<<<h->sm_count * 8, 256, 0, h->stream>>>(cap, h->ft_keys.as<unsigned long long>(), h->ft_cnt.as<unsigned>(),
                                                    h->colmin.as<unsigned>());
  LAUNCH_CHECK(h);
  oa_colbase<<<cdiv(M1, OA_THREADS), OA_THREADS, 0, h->stream>>>(M1, h->colmin.as<unsigned>(), h->colmax.as<unsigned>(),
                                                                 ls.cur + r);
  LAUNCH_CHECK(h);
  oa_expand<<<cdiv((long long)cap, OA_THREADS), OA_THREADS, 0, h->stream>>>(
      cap, h->ft_keys.as<unsigned long long>(), h->ft_cnt.as<unsigned>(), h->colmax.as<unsigned>(), (size_t)M1, lv.keys,
      lv.cnt, ls.cur + r, lv.colcnt, lv.diag, h->scalars.as<DevScalars>());
  LAUNCH_CHECK(h);
  return GK_OK;
}

// Reads the levels' column statistics back (synchronises) into the handle's per-level tables.
static int level_finish(gk_handle* h, const LevelScratch& ls, int n_blocks, const char* who, DevScalars** hs,
                        int64_t* n_cols, int64_t* n_ent) {
  GK_CUDA(cudaMemcpyAsync(h->h_colstats.p, h->nh_cur.p, ls.cur_bytes, cudaMemcpyDeviceToHost, h->stream));
  GK_TRY(read_scalars(h, hs));  // synchronises
  if ((*hs)->ft_overflow) return fail(GK_ERR_STATE, std::string(who) + ": expanded feature block overflow");
  const OaCursors* hc = h->h_colstats.as<OaCursors>();
  const unsigned long long* hdims = reinterpret_cast<const unsigned long long*>(hc + n_blocks);
  h->nh_dims.assign(n_blocks, 0);
  h->nh_cols.assign(n_blocks, 0);
  h->nh_entries.assign(n_blocks, 0);
  *n_cols = *n_ent = 0;
  for (int r = 0; r < n_blocks; ++r) {
    h->nh_dims[r] = (long long)hdims[r];
    h->nh_cols[r] = (long long)hc[r].n_cols;
    h->nh_entries[r] = (long long)hc[r].n_entries;
    *n_cols += h->nh_cols[r];
    *n_ent += h->nh_entries[r];
  }
  return GK_OK;
}

int gk_nh_features(gk_handle* h, int32_t R, int32_t nh_type, int32_t bits, const uint64_t* code_of_label,
                   const uint8_t* label_valid, int64_t n_labels, int32_t flags, gk_stats* stats) {
  GK_TRY(need_packed(h, "gk_nh_features"));
  if (!h->has_labels) return fail(GK_ERR_ARG, "gk_nh_features: vertex labels are required");
  if (R < 1 || R > MAX_LEVELS) return fail(GK_ERR_ARG, "gk_nh_features: R out of range [1, 64]");
  if (nh_type != GK_NH_SIMPLE && nh_type != GK_NH_COUNT_SENSITIVE) return fail(GK_ERR_ARG, "gk_nh_features: unknown nh_type");
  if (bits < 1 || bits > 64) return fail(GK_ERR_ARG, "gk_nh_features: bits out of range [1, 64]");
  if (flags != 0) return fail(GK_ERR_ARG, "gk_nh_features: no flags are defined");
  if (!code_of_label || n_labels < h->n_labels0) return fail(GK_ERR_ARG, "gk_nh_features: a code is needed for every label id");
  const int64_t N = h->N, V = h->V, E = h->E;
  const int64_t V1 = std::max<int64_t>(V, 1), L1 = std::max<int64_t>(n_labels, 1);
  const unsigned long long mask = bits == 64 ? ~0ULL : (1ULL << bits) - 1ULL;
  const int64_t launches0 = h->launches;
  features_begin(h);

  GK_TRY(init_scalars(h, 0));  // clears ft_overflow
  GK_TRY(h->nh_codes.ensure((size_t)(R + 1) * V1 * 8));
  GK_TRY(h->nh_valid.ensure((size_t)(R + 1) * V1));
  GK_TRY(h->nh_lut.ensure((size_t)L1 * 9));
  unsigned long long* codes = h->nh_codes.as<unsigned long long>();
  unsigned char* valid = h->nh_valid.as<unsigned char>();
  unsigned char* d_lvalid = h->nh_lut.as<unsigned char>() + (size_t)L1 * 8;
  if (n_labels > 0) {
    GK_CUDA(cudaMemcpyAsync(h->nh_lut.p, code_of_label, (size_t)n_labels * 8, cudaMemcpyHostToDevice, h->stream));
    if (label_valid) GK_CUDA(cudaMemcpyAsync(d_lvalid, label_valid, (size_t)n_labels, cudaMemcpyHostToDevice, h->stream));
    else GK_CUDA(cudaMemsetAsync(d_lvalid, 1, (size_t)n_labels, h->stream));
  }
  // count-sensitive tables of the large-degree vertices: 2 slots per edge
  // (2 E slots: row position | count | two-codes flag)
  if (nh_type == GK_NH_COUNT_SENSITIVE && h->n_large) GK_TRY(h->nh_ws.ensure((size_t)std::max<int64_t>(E, 1) * 24));
  GK_CUDA(cudaEventRecord(h->tev[2], h->stream));

  // ---- hash levels: gr[0] = NH(initial), gr[r] = NH(gr[r - 1])
  if (V) {
    nh_init<<<cdiv(V, 256), 256, 0, h->stream>>>((int)V, h->labels0.as<int>(), h->nh_lut.as<unsigned long long>(), d_lvalid,
                                                 codes, valid);
    LAUNCH_CHECK(h);
  }
  int* ws_tab = h->nh_ws.as<int>();
  unsigned* ws_cnt = reinterpret_cast<unsigned*>(ws_tab + 2 * std::max<int64_t>(E, 1));
  unsigned* order_dep = &h->scalars.as<DevScalars>()->nh_order_dep;
  for (int r = 0; r < R && V; ++r) {
    const unsigned long long* in = codes + (size_t)r * V;
    const unsigned char* vin = valid + (size_t)r * V;
    unsigned long long* out = codes + (size_t)(r + 1) * V;
    unsigned char* vout = valid + (size_t)(r + 1) * V;
    if (nh_type == GK_NH_SIMPLE)
      nh_hash_small<NH_SIMPLE><<<cdiv(V, 256), 256, 0, h->stream>>>((int)V, h->group_width, h->row_ptr.as<int>(),
                                                                    h->col_idx.as<int>(), in, vin, out, vout, bits, mask, order_dep);
    else
      nh_hash_small<NH_COUNT><<<cdiv(V, 256), 256, 0, h->stream>>>((int)V, h->group_width, h->row_ptr.as<int>(),
                                                                   h->col_idx.as<int>(), in, vin, out, vout, bits, mask, order_dep);
    LAUNCH_CHECK(h);
    if (h->n_large) {  // vertices of degree > group_width (gk_pack_csr's large list)
      if (nh_type == GK_NH_SIMPLE)
        nh_hash_large<NH_SIMPLE><<<(int)h->n_large, NH_LARGE_THREADS, 0, h->stream>>>(
            h->large_list.as<int>(), h->row_ptr.as<int>(), h->col_idx.as<int>(), in, vin, out, vout, bits, mask, nullptr, nullptr, order_dep);
      else
        nh_hash_large<NH_COUNT><<<(int)h->n_large, NH_LARGE_THREADS, 0, h->stream>>>(
            h->large_list.as<int>(), h->row_ptr.as<int>(), h->col_idx.as<int>(), in, vin, out, vout, bits, mask, ws_tab, ws_cnt, order_dep);
      LAUNCH_CHECK(h);
    }
  }
  GK_CUDA(cudaEventRecord(h->tev[5], h->stream));

  // ---- per-level columns, counts and unary expansion
  LevelScratch ls;
  GK_TRY(level_setup(h, V, R, &ls));
  for (int r = 0; r < R; ++r)
    GK_TRY(level_columns(h, ls, r, V, 1, codes + (size_t)(r + 1) * V, valid + (size_t)(r + 1) * V));
  GK_CUDA(cudaEventRecord(h->tev[3], h->stream));
  DevScalars* hs;
  int64_t n_cols = 0, n_ent = 0;
  GK_TRY(level_finish(h, ls, R, "gk_nh_features", &hs, &n_cols, &n_ent));
  h->nh_R = R;
  h->n_columns = n_cols;
  features_publish(h, FK_NH);
  if (stats) {
    memset(stats, 0, sizeof(*stats));
    stats->n_graphs = N; stats->n_vertices = V; stats->n_edges = E;
    stats->n_levels = R;
    for (int r = 0; r < R; ++r) stats->level_dims[r] = h->nh_dims[r];
    stats->n_columns = n_cols;
    stats->n_entries = n_ent;
    stats->kernel_launches = h->launches - launches0;
    stats->ms_features = ev_ms(h->tev[2], h->tev[3]);
    stats->ms_hash = ev_ms(h->tev[2], h->tev[5]);
    stats->ms_columns = ev_ms(h->tev[5], h->tev[3]);
    stats->nh_order_dependent = hs->nh_order_dep ? 1 : 0;
  }
  return GK_OK;
}

int gk_nh_labels(gk_handle* h, int32_t level, uint64_t* out, uint8_t* valid) {
  if (!h || !out) return fail(GK_ERR_ARG, "gk_nh_labels: null argument");
  if (h->feature_kind != FK_NH || level < 0 || level >= h->nh_R)
    return fail(GK_ERR_STATE, "gk_nh_labels: no such level (run gk_nh_features first)");
  GK_CUDA(cudaSetDevice(h->dev));
  const size_t V = (size_t)h->V;
  if (V) {
    GK_CUDA(cudaMemcpyAsync(out, h->nh_codes.as<unsigned long long>() + (size_t)(level + 1) * V, V * 8,
                            cudaMemcpyDeviceToHost, h->stream));
    if (valid)
      GK_CUDA(cudaMemcpyAsync(valid, h->nh_valid.as<unsigned char>() + (size_t)(level + 1) * V, V, cudaMemcpyDeviceToHost,
                              h->stream));
    GK_CUDA(cudaStreamSynchronize(h->stream));
  }
  return GK_OK;
}

// The per-level Gram driver of NeighborhoodHash (gram_path 7) and PyramidMatch (gram_path 11): for every one of the
// n_blocks level blocks, gram_int's exact integer Gram of the block gives the intersection counts as fp32 in nh_C;
// `combine` turns the n_blocks count matrices of a row chunk into the fp64 K.  Rows go in chunks when the count
// matrices of the whole request would exceed LEVEL_C_BUDGET bytes (GRAKEL_B200_NH_C_BUDGET=<bytes> lowers it, so that
// tests reach the chunked route; a chunk of the square case then computes full rows instead of mirroring).
}  // extern "C" (a template driver follows)

constexpr size_t LEVEL_C_BUDGET = (size_t)8 << 30;

struct LevelChunk {  // what a combine kernel reads and writes for rows [cb, cb + rows) of the request
  const float* C;    // n_blocks matrices [rows x ldc], block r at C + r * stride
  long long stride, ldc;
  int row_g0;        // packed graph of the chunk's first row
  int rows, cols;
  int mirror;        // the full square matrix: compute upper tiles and mirror them
  double* out;
  long long ld;
};

struct LevelTimes {
  std::vector<float> ms_block;
  float ms_combine = 0.f;
  int64_t max_T = 0, gram_launches = 0, elem_bytes = 0;
};

template <class Combine>
static int gram_levels(gk_handle* h, const GramReq& q, int n_blocks, const F64Out& out, Combine combine, LevelTimes* t) {
  const int64_t N = h->N, n_fit = q.n_fit, k_rows = q.k_rows, k_cols = q.k_cols;
  const bool square = q.square;
  const int64_t ldc = (k_cols + 7) / 8 * 8;  // 32-byte rows: TMA stores of the Gram epilogue
  size_t c_budget = LEVEL_C_BUDGET;
  if (const char* e = getenv("GRAKEL_B200_NH_C_BUDGET")) c_budget = std::max<size_t>(1, strtoull(e, nullptr, 10));
  const int64_t chunk = std::max<int64_t>(1, std::min<int64_t>(std::max<int64_t>(k_rows, 1),
                                                                (int64_t)(c_budget / ((size_t)n_blocks * ldc * 4))));
  GK_TRY(h->nh_C.ensure((size_t)n_blocks * chunk * ldc * 4));
  const int32_t gflags = (q.flags & (GK_GRAM_SIMT | GK_DENSE_ALL | GK_FULL_TILES)) | GK_OUT_DEVICE;
  GK_TRY(h->part_max.ensure(4));
  GK_TRY(h->part_new.ensure(4));
  t->ms_block.assign(n_blocks, 0.f);
  gk_stats st;
  for (int64_t cb = q.row_begin; cb < q.row_end; cb += chunk) {
    const int64_t ce = std::min<int64_t>(q.row_end, cb + chunk), rows = ce - cb;
    for (int r = 0; r < n_blocks; ++r) {
      // the integer Gram of level block r: its rows [cb, ce) as fp32 counts into nh_C
      IntBlock fb = nh_level(h, r);
      fb.n_columns = h->nh_cols[r];
      const unsigned part[2] = {h->nh_entries[r] ? 1u : 0u, (unsigned)h->nh_entries[r]};
      GK_CUDA(cudaMemcpyAsync(h->part_max.p, &part[0], 4, cudaMemcpyHostToDevice, h->stream));
      GK_CUDA(cudaMemcpyAsync(h->part_new.p, &part[1], 4, cudaMemcpyHostToDevice, h->stream));
      GramReq lq;
      GK_TRY(gram_request(h, FK_WL, n_fit, gflags, cb, ce, h->nh_C.as<float>() + (size_t)r * chunk * ldc, GK_F32, ldc,
                          nullptr, nullptr, &lq));
      memset(&st, 0, sizeof(st));
      GK_TRY(gram_int(h, lq, fb, &st));
      t->ms_block[r] += st.ms_total;
      t->max_T = std::max<int64_t>(t->max_T, st.threshold);
      t->gram_launches += st.gemm_launches;
      t->elem_bytes = std::max<int64_t>(t->elem_bytes, st.gemm_elem_bytes);  // 0 when no tensor-core GEMM ran
    }
    if (rows > 0) {
      LevelChunk c;
      c.C = h->nh_C.as<float>();
      c.stride = chunk * ldc;
      c.ldc = ldc;
      c.row_g0 = (int)((square ? 0 : n_fit) + cb);
      c.rows = (int)rows;
      c.cols = (int)k_cols;
      c.mirror = square && cb == 0 && ce == N && !(q.flags & GK_FULL_TILES) ? 1 : 0;
      c.out = out.p + (size_t)(cb - q.row_begin) * out.ld;
      c.ld = out.ld;
      GK_CUDA(cudaEventRecord(h->tev[0], h->stream));
      GK_TRY(combine(c));
      GK_CUDA(cudaEventRecord(h->tev[1], h->stream));
      GK_CUDA(cudaEventSynchronize(h->tev[1]));
      t->ms_combine += ev_ms(h->tev[0], h->tev[1]);
    }
  }
  return GK_OK;
}

extern "C" {

// Gram of NeighborhoodHash features (gram_path 7): gram_levels with nh_combine.  GK_NORMALIZE changes nothing: the
// reference never normalises this kernel, and its self similarities are 1.
static int gram_nh(gk_handle* h, const GramReq& q, gk_stats* stats) {
  const int64_t N = h->N, n_fit = q.n_fit, k_cols = q.k_cols;
  const int R = h->nh_R;
  const bool square = q.square;
  const int64_t launches0 = h->launches;
  F64Out out;
  GK_TRY(f64_target(h, q, &out));
  LevelTimes lt;
  GK_TRY(gram_levels(h, q, R, out, [&](const LevelChunk& c) {
    NhCombineParams p;
    p.C = c.C;
    p.stride = c.stride;
    p.ldc = c.ldc;
    p.R = R;
    p.graph_ptr = h->graph_ptr.as<int>();
    p.row_g0 = c.row_g0;
    p.rows = c.rows;
    p.cols = c.cols;
    p.mirror = c.mirror;
    p.out = c.out;
    p.ld = c.ld;
    const long long nbi = (c.rows + NH_TILE - 1) / NH_TILE, nbj = (k_cols + NH_TILE - 1) / NH_TILE;
    const long long grid = p.mirror ? nbj * (nbj + 1) / 2 : nbi * nbj;
    if (grid > 0) {
      nh_combine<<<(unsigned)grid, NH_TILE * 8, 0, h->stream>>>(p);
      LAUNCH_CHECK(h);
    }
    return GK_OK;
  }, &lt));
  const float ms_combine = lt.ms_combine;
  GramReq kq = q;  // the self similarities are 1, written on the host
  kq.xdiag = kq.ydiag = nullptr;
  GK_TRY(f64_deliver(h, kq, out, false, h->ev[14], h->ev[15]));
  if (q.xdiag) for (int64_t i = 0; i < n_fit; ++i) q.xdiag[i] = 1.0;
  if (q.ydiag && !square) for (int64_t i = 0; i < N - n_fit; ++i) q.ydiag[i] = 1.0;
  if (stats) {
    stats->n_graphs = N; stats->n_vertices = h->V; stats->n_edges = h->E;
    stats->n_levels = R;
    stats->gram_path = 7;
    stats->threshold = lt.max_T;
    stats->max_count = 1;
    stats->gemm_launches = lt.gram_launches + (h->launches - launches0);
    stats->gemm_elem_bytes = lt.elem_bytes;
    float tot = ms_combine;
    for (int r = 0; r < R; ++r) { stats->ms_level_gram[r] = lt.ms_block[r]; tot += lt.ms_block[r]; }
    stats->ms_gemm = tot - ms_combine;
    stats->ms_combine = ms_combine;
    stats->ms_d2h = ev_ms(h->ev[14], h->ev[15]);
    stats->ms_total = tot + stats->ms_d2h;
  }
  return GK_OK;
}

// ---------------------------------------------------------------------------
// PyramidMatch (pyramid_match.cuh).  The host hands over n_sets embedding sets U [n_sets][V][d] fp64 (|U| of every
// vertex, zero past its graph's column count) and the column counts [n_sets][N]; each set's L levels become level
// blocks s * L + j of the NeighborhoodHash layout.  Histogram rows come from the packed label ids (GK_PM_LABELS), from
// WL level s of a preceding gk_wl_features (GK_PM_WL_LABELS: one set per WL level) or are the dimension alone.
static int pm_keys(gk_handle* h, int s, int j, unsigned long long* keys, unsigned char* valid) {
  const int64_t V = h->V, N = h->N, M = V * h->pm_d;
  if (!M) return GK_OK;
  const int* labels = nullptr;
  if (h->pm_flags & GK_PM_WL_LABELS) labels = h->labels_all.as<int>() + (size_t)s * V;
  else if (h->pm_flags & GK_PM_LABELS) labels = h->labels0.as<int>();
  pm_cells<<<cdiv(M, 256), 256, 0, h->stream>>>((int)M, h->pm_d, j, h->pm_U.as<double>() + (size_t)s * M,
                                                h->pm_ncols.as<int>() + (size_t)s * N, h->vgraph.as<int>(), labels,
                                                h->pm_has_skip ? h->pm_skip.as<unsigned char>() : nullptr, keys, valid);
  LAUNCH_CHECK(h);
  return GK_OK;
}

int gk_pm_features(gk_handle* h, int32_t n_iter, int32_t L, int32_t d, const double* U, const int32_t* n_cols,
                   const uint8_t* skip, int32_t n_sets, int32_t flags, gk_stats* stats) {
  GK_TRY(need_packed(h, "gk_pm_features"));
  if (L < 0) return fail(GK_ERR_ARG, "gk_pm_features: L < 0");
  if (L > MAX_LEVELS) return fail(GK_ERR_UNSUPPORTED, "gk_pm_features: at most L = 64 levels are supported");
  if (d < 1 || n_sets < 1) return fail(GK_ERR_ARG, "gk_pm_features: d and n_sets must be positive");
  if (flags & ~(GK_PM_LABELS | GK_PM_WL_LABELS)) return fail(GK_ERR_ARG, "gk_pm_features: unknown flags");
  if (!n_cols || (!U && h->V)) return fail(GK_ERR_ARG, "gk_pm_features: null embeddings or column counts");
  const bool wl = flags & GK_PM_WL_LABELS;
  if (wl && (h->feature_kind != FK_WL || h->n_levels != n_iter + 1 || n_sets != n_iter + 1))
    return fail(GK_ERR_STATE, "gk_pm_features: GK_PM_WL_LABELS needs gk_wl_features(n_iter) first and n_iter + 1 sets");
  if (!wl && n_sets != 1 && (flags & GK_PM_LABELS)) return fail(GK_ERR_ARG, "gk_pm_features: one set per label source");
  if ((flags & GK_PM_LABELS) && !wl && !h->has_labels) return fail(GK_ERR_ARG, "gk_pm_features: vertex labels are required");
  const int64_t N = h->N, V = h->V, M = V * (int64_t)d;
  if (M >= (1LL << 31)) return fail(GK_ERR_UNSUPPORTED, "gk_pm_features: V * d must stay below 2^31");
  // the level Grams count in fp32: exact while every intersection (<= d * n_max) stays below 2^24
  if ((int64_t)h->max_graph_size * d >= (1LL << 24))
    return fail(GK_ERR_UNSUPPORTED, "gk_pm_features: d * (largest graph) must stay below 2^24");
  // (row, cell) keys: row < n_lab * d, cell < 2^(L-1), row << (L-1) must fit 64 bits
  const int64_t n_lab = wl ? std::max<int64_t>(h->n_labels0, V) : (flags & GK_PM_LABELS) ? h->n_labels0 : 1;
  if (L > 0) {
    const unsigned long long rows = (unsigned long long)std::max<int64_t>(n_lab, 1) * (unsigned long long)d;
    int bits = 0;
    while (bits < 64 && (rows - 1) >> bits) ++bits;
    if (bits + (L - 1) > 64) return fail(GK_ERR_UNSUPPORTED, "gk_pm_features: a (histogram row, cell) key does not fit 64 bits");
  }
  for (int64_t i = 0; i < (int64_t)n_sets * N; ++i)
    if (n_cols[i] < 0 || n_cols[i] > d) return fail(GK_ERR_ARG, "gk_pm_features: a column count is outside [0, d]");
  // every used u must lie in [0, 1 + 2^-(L-1)): a NaN or negative u has no cell, and a larger one would give a cell
  // past the clamp 2^j - 1 that runs into the next row's keys
  if (L > 0 && V) {
    const std::vector<int>& gp = h->graph_ptr_host;
    const double top = ldexp(1.0, L - 1);
    for (int s = 0; s < n_sets; ++s)
      for (int64_t g = 0; g < N; ++g)
        for (int64_t v = gp[g]; v < gp[g + 1]; ++v) {
          if (skip && skip[v]) continue;
          const double* u = U + ((size_t)s * V + v) * d;
          for (int q = 0; q < n_cols[(size_t)s * N + g]; ++q)
            if (!(u[q] >= 0.0) || floor(u[q] * top) > top)
              return fail(GK_ERR_ARG, "gk_pm_features: an embedding value is NaN, negative or >= 1 + 2^-(L-1)");
        }
  }
  const int64_t launches0 = h->launches;
  features_begin(h);
  GK_TRY(init_scalars(h, 0));  // clears ft_overflow
  GK_CUDA(cudaEventRecord(h->tev[2], h->stream));
  if (wl && h->wl_sparse_ids) {  // the histogram rows are indexed by dense label ids
    for (int lv = 1; lv <= n_iter; ++lv) GK_TRY(wl_densify(h, lv, h->labels_all.as<int>() + (size_t)lv * V));
    h->wl_sparse_ids = false;
  }
  GK_TRY(h->pm_U.ensure((size_t)n_sets * std::max<int64_t>(M, 1) * 8));
  GK_TRY(h->pm_ncols.ensure((size_t)n_sets * N * 4));
  if (M) GK_CUDA(cudaMemcpyAsync(h->pm_U.p, U, (size_t)n_sets * M * 8, cudaMemcpyHostToDevice, h->stream));
  GK_CUDA(cudaMemcpyAsync(h->pm_ncols.p, n_cols, (size_t)n_sets * N * 4, cudaMemcpyHostToDevice, h->stream));
  h->pm_has_skip = skip != nullptr && V > 0;
  if (h->pm_has_skip) {
    GK_TRY(h->pm_skip.ensure((size_t)V));
    GK_CUDA(cudaMemcpyAsync(h->pm_skip.p, skip, (size_t)V, cudaMemcpyHostToDevice, h->stream));
  }
  h->pm_S = n_sets; h->pm_L = L; h->pm_d = d; h->pm_flags = flags;
  const int n_blocks = n_sets * L;
  GK_TRY(h->nh_codes.ensure((size_t)std::max<int64_t>(M, 1) * 8));
  GK_TRY(h->nh_valid.ensure((size_t)std::max<int64_t>(M, 1)));
  unsigned long long* keys = h->nh_codes.as<unsigned long long>();
  unsigned char* valid = h->nh_valid.as<unsigned char>();
  LevelScratch ls;
  GK_TRY(level_setup(h, M, std::max(n_blocks, 1), &ls));
  for (int s = 0; s < n_sets; ++s)
    for (int j = 0; j < L; ++j) {
      GK_TRY(pm_keys(h, s, j, keys, valid));
      GK_TRY(level_columns(h, ls, s * L + j, M, d, keys, valid));
    }
  GK_CUDA(cudaEventRecord(h->tev[3], h->stream));
  DevScalars* hs;
  int64_t n_col = 0, n_ent = 0;
  GK_TRY(level_finish(h, ls, n_blocks, "gk_pm_features", &hs, &n_col, &n_ent));
  h->nh_R = n_blocks;
  h->n_columns = n_col;
  features_publish(h, FK_PM);
  if (stats) {
    memset(stats, 0, sizeof(*stats));
    stats->n_graphs = N; stats->n_vertices = V; stats->n_edges = h->E;
    stats->n_levels = n_blocks;
    for (int r = 0; r < std::min(n_blocks, MAX_LEVELS); ++r) stats->level_dims[r] = h->nh_dims[r];
    stats->n_columns = n_col;
    stats->n_entries = n_ent;
    stats->kernel_launches = h->launches - launches0;
    stats->ms_features = ev_ms(h->tev[2], h->tev[3]);
    stats->ms_columns = stats->ms_features;
  }
  return GK_OK;
}

int gk_pm_cells(gk_handle* h, int32_t set, int32_t level, int64_t* out) {
  if (!h || !out) return fail(GK_ERR_ARG, "gk_pm_cells: null argument");
  if (h->feature_kind != FK_PM || set < 0 || set >= h->pm_S || level < 0 || level >= h->pm_L)
    return fail(GK_ERR_STATE, "gk_pm_cells: no such set / level (run gk_pm_features first)");
  GK_CUDA(cudaSetDevice(h->dev));
  const size_t M = (size_t)h->V * h->pm_d;
  if (!M) return GK_OK;
  // the level's keys are recomputed into the scratch of gk_pm_features (its level blocks are not touched)
  GK_TRY(pm_keys(h, set, level, h->nh_codes.as<unsigned long long>(), h->nh_valid.as<unsigned char>()));
  std::vector<unsigned long long> keys(M);
  std::vector<unsigned char> valid(M);
  GK_CUDA(cudaMemcpyAsync(keys.data(), h->nh_codes.p, M * 8, cudaMemcpyDeviceToHost, h->stream));
  GK_CUDA(cudaMemcpyAsync(valid.data(), h->nh_valid.p, M, cudaMemcpyDeviceToHost, h->stream));
  GK_CUDA(cudaStreamSynchronize(h->stream));
  const unsigned long long mask = level == 0 ? 0ULL : (level >= 64 ? ~0ULL : (1ULL << level) - 1ULL);
  for (size_t e = 0; e < M; ++e) out[e] = valid[e] ? (int64_t)(keys[e] & mask) : -1;
  return GK_OK;
}

// Gram of PyramidMatch features (gram_path 11): gram_levels with pm_combine; self similarities from pm_diag, so
// GK_NORMALIZE divides by sqrt(K_ii K_jj) as the reference's base class does.
static int gram_pm(gk_handle* h, const GramReq& q, gk_stats* stats) {
  const int64_t N = h->N, k_cols = q.k_cols;
  const int S = h->pm_S, L = h->pm_L, n_blocks = S * L;
  const int64_t launches0 = h->launches;
  F64Out out;
  GK_TRY(f64_target(h, q, &out));
  LevelTimes lt;
  if (n_blocks == 0) {  // L = 0: the reference's k stays 0
    if (q.k_rows > 0) GK_CUDA(cudaMemset2DAsync(out.p, (size_t)out.ld * 8, 0, (size_t)k_cols * 8, (size_t)q.k_rows, h->stream));
  } else {
    GK_TRY(gram_levels(h, q, n_blocks, out, [&](const LevelChunk& c) {
      PmCombineParams p;
      p.C = c.C;
      p.stride = c.stride;
      p.ldc = c.ldc;
      p.S = S;
      p.L = L;
      p.rows = c.rows;
      p.cols = c.cols;
      p.mirror = c.mirror;
      p.out = c.out;
      p.ld = c.ld;
      const long long nbi = (c.rows + PM_TILE - 1) / PM_TILE, nbj = (k_cols + PM_TILE - 1) / PM_TILE;
      const long long grid = p.mirror ? nbj * (nbj + 1) / 2 : nbi * nbj;
      if (grid > 0) {
        pm_combine<<<(unsigned)grid, PM_TILE * 8, 0, h->stream>>>(p);
        LAUNCH_CHECK(h);
      }
      return GK_OK;
    }, &lt));
  }
  // after the level Grams: gram_int leaves each level block's own self similarities in diag_f64
  GK_TRY(h->diag_f64.ensure((size_t)N * 8));
  pm_diag<<<cdiv(N, 256), 256, 0, h->stream>>>((int)N, S, L, h->graph_ptr.as<int>(), h->pm_ncols.as<int>(),
                                               h->pm_has_skip ? h->pm_skip.as<unsigned char>() : nullptr,
                                               h->diag_f64.as<double>());
  LAUNCH_CHECK(h);
  GK_TRY(f64_deliver(h, q, out, true, h->ev[14], h->ev[15]));
  if (stats) {
    stats->n_graphs = N; stats->n_vertices = h->V; stats->n_edges = h->E;
    stats->n_levels = L;
    stats->gram_path = 11;
    stats->threshold = lt.max_T;
    stats->max_count = 1;
    stats->gemm_launches = lt.gram_launches + (h->launches - launches0);
    stats->gemm_elem_bytes = lt.elem_bytes;
    float tot = lt.ms_combine;
    for (int j = 0; j < L; ++j) stats->ms_level_gram[j] = 0.f;
    for (int r = 0; r < n_blocks; ++r) { stats->ms_level_gram[r % L] += lt.ms_block[r]; tot += lt.ms_block[r]; }
    stats->ms_gemm = tot - lt.ms_combine;
    stats->ms_combine = lt.ms_combine;
    stats->ms_d2h = ev_ms(h->ev[14], h->ev[15]);
    stats->ms_total = tot + stats->ms_d2h;
  }
  return GK_OK;
}

// ---------------------------------------------------------------------------
// Random walk kernels (random_walk.cuh).  gk_rw_features uploads what the route reads; gk_gram (gram_rw) runs one CTA
// per graph pair.
int gk_rw_features(gk_handle* h, int32_t route, int32_t fn, double lamda, const double* coef, int32_t n_coef,
                   const double* values, const int32_t* t_row_ptr, const int32_t* t_col_idx, const double* t_values,
                   const double* q, const double* w, int32_t flags, gk_stats* stats) {
  GK_TRY(need_packed(h, "gk_rw_features"));
  if (route != GK_RW_CG && route != GK_RW_SPECTRAL && route != GK_RW_SERIES) return fail(GK_ERR_ARG, "gk_rw_features: unknown route");
  if (fn != GK_RW_FINITE && fn != GK_RW_EXP && fn != GK_RW_INV) return fail(GK_ERR_ARG, "gk_rw_features: unknown fn");
  if (flags & ~GK_RW_LABELED) return fail(GK_ERR_ARG, "gk_rw_features: unknown flags");
  if ((flags & GK_RW_LABELED) && !h->has_labels) return fail(GK_ERR_ARG, "gk_rw_features: GK_RW_LABELED needs packed labels");
  if (fn == GK_RW_FINITE && (!coef || n_coef < 1)) return fail(GK_ERR_ARG, "gk_rw_features: the finite series needs coefficients");
  if (route == GK_RW_SPECTRAL && (!q || !w)) return fail(GK_ERR_ARG, "gk_rw_features: the spectral route needs q and w");
  if (route == GK_RW_SPECTRAL && (flags & GK_RW_LABELED)) return fail(GK_ERR_UNSUPPORTED, "gk_rw_features: no labelled spectral route");
  if (route == GK_RW_CG && fn != GK_RW_INV) return fail(GK_ERR_ARG, "gk_rw_features: conjugate gradients solve the geometric kernel (GK_RW_INV)");
  if (route == GK_RW_SERIES && fn == GK_RW_INV) return fail(GK_ERR_UNSUPPORTED, "gk_rw_features: no series for the geometric inverse");
  if (route != GK_RW_SPECTRAL && h->E > 0 && (!values || !t_row_ptr || !t_col_idx || !t_values))
    return fail(GK_ERR_ARG, "gk_rw_features: edge values and the transposed CSR are required");
  const int64_t V = h->V, E = h->E;
  if (route != GK_RW_SPECTRAL && t_row_ptr && (t_row_ptr[0] != 0 || t_row_ptr[V] != E))
    return fail(GK_ERR_ARG, "gk_rw_features: transposed row_ptr does not match the packed block");
  features_begin(h);
  GK_CUDA(cudaEventRecord(h->tev[0], h->stream));
  if (route != GK_RW_SPECTRAL) {
    GK_TRY(h->rw_val.ensure(std::max<int64_t>(E, 1) * 8));
    GK_TRY(h->rw_tval.ensure(std::max<int64_t>(E, 1) * 8));
    GK_TRY(h->rw_tci.ensure(std::max<int64_t>(E, 1) * 4));
    GK_TRY(h->rw_trp.ensure((V + 1) * 4));
    if (t_row_ptr) {
      GK_CUDA(cudaMemcpyAsync(h->rw_trp.p, t_row_ptr, (V + 1) * 4, cudaMemcpyHostToDevice, h->stream));
    } else {
      GK_CUDA(cudaMemsetAsync(h->rw_trp.p, 0, (V + 1) * 4, h->stream));
    }
    if (E) {
      GK_CUDA(cudaMemcpyAsync(h->rw_val.p, values, E * 8, cudaMemcpyHostToDevice, h->stream));
      GK_CUDA(cudaMemcpyAsync(h->rw_tval.p, t_values, E * 8, cudaMemcpyHostToDevice, h->stream));
      GK_CUDA(cudaMemcpyAsync(h->rw_tci.p, t_col_idx, E * 4, cudaMemcpyHostToDevice, h->stream));
    }
  } else {
    GK_TRY(h->rw_q.ensure(std::max<int64_t>(V, 1) * 8));
    GK_TRY(h->rw_w.ensure(std::max<int64_t>(V, 1) * 8));
    if (V) {
      GK_CUDA(cudaMemcpyAsync(h->rw_q.p, q, V * 8, cudaMemcpyHostToDevice, h->stream));
      GK_CUDA(cudaMemcpyAsync(h->rw_w.p, w, V * 8, cudaMemcpyHostToDevice, h->stream));
    }
  }
  h->rw_ncoef = fn == GK_RW_FINITE ? n_coef : 0;
  if (h->rw_ncoef) {
    GK_TRY(h->rw_coef.ensure((size_t)n_coef * 8));
    GK_CUDA(cudaMemcpyAsync(h->rw_coef.p, coef, (size_t)n_coef * 8, cudaMemcpyHostToDevice, h->stream));
  }
  GK_TRY(h->rw_cap.ensure(8));
  GK_CUDA(cudaEventRecord(h->tev[1], h->stream));
  GK_CUDA(cudaStreamSynchronize(h->stream));  // the caller's buffers may be reused once we return
  h->rw_route = route; h->rw_fn = fn; h->rw_lamda = lamda;
  h->rw_labeled = (flags & GK_RW_LABELED) != 0;
  features_publish(h, FK_RW);
  if (stats) {
    stats->n_graphs = h->N; stats->n_vertices = V; stats->n_edges = E;
    stats->ms_h2d = ev_ms(h->tev[0], h->tev[1]);
  }
  return GK_OK;
}

int gk_rw_iterations(gk_handle* h, uint8_t* out) {
  if (!h || !out) return fail(GK_ERR_ARG, "gk_rw_iterations: null argument");
  if (h->feature_kind != FK_RW || h->rw_iter_rows * h->rw_iter_cols == 0) return fail(GK_ERR_STATE, "gk_rw_iterations: no random walk Gram yet");
  GK_CUDA(cudaSetDevice(h->dev));
  GK_CUDA(cudaMemcpyAsync(out, h->rw_iters.p, (size_t)(h->rw_iter_rows * h->rw_iter_cols), cudaMemcpyDeviceToHost, h->stream));
  GK_CUDA(cudaStreamSynchronize(h->stream));
  return GK_OK;
}

// ---------------------------------------------------------------------------
// Propagation (propagation.cuh).  The packed CSR is the sparsity pattern of the row-normalised transition matrices,
// t_values[E] their entries; the features are the SP layout (FK_PK), so gk_gram's integer route runs them.
int gk_pk_features(gk_handle* h, int32_t t_max, double w, const double* u, const double* b, int32_t dim,
                   int32_t dim_orig, int64_t n_fit, const double* t_values, const double* p0, int32_t flags,
                   gk_stats* stats) {
  GK_TRY(need_packed(h, "gk_pk_features"));
  if (t_max < 1 || t_max > MAX_LEVELS) return fail(GK_ERR_ARG, "gk_pk_features: t_max out of range [1, 64]");
  if (!(w != 0.0) || !std::isfinite(w)) return fail(GK_ERR_ARG, "gk_pk_features: w must be finite and non-zero");
  if (flags & ~(GK_PK_ATTR | GK_PK_SQRT | GK_PK_STORE_F32 | GK_PK_STORE_INT | GK_PK_NEW_LABELS))
    return fail(GK_ERR_ARG, "gk_pk_features: unknown flag");
  const bool attr = flags & GK_PK_ATTR, split = flags & GK_PK_NEW_LABELS;
  if ((flags & GK_PK_STORE_F32) && (flags & GK_PK_STORE_INT)) return fail(GK_ERR_ARG, "gk_pk_features: two storage modes");
  if (attr && (split || (flags & GK_PK_SQRT))) return fail(GK_ERR_ARG, "gk_pk_features: GK_PK_SQRT / GK_PK_NEW_LABELS are for labels");
  if (!attr && (flags & (GK_PK_STORE_F32 | GK_PK_STORE_INT))) return fail(GK_ERR_ARG, "gk_pk_features: storage modes are for attributes");
  if (dim < 1 || dim_orig < 0 || dim_orig > dim || (!split && dim_orig != dim))
    return fail(GK_ERR_ARG, "gk_pk_features: bad dim / dim_orig");
  if (n_fit < 0 || n_fit > h->N) return fail(GK_ERR_ARG, "gk_pk_features: n_fit out of range");
  if (!u || !b || (h->E && !t_values)) return fail(GK_ERR_ARG, "gk_pk_features: null argument");
  if (attr && !p0 && h->V) return fail(GK_ERR_ARG, "gk_pk_features: attributes need p0");
  if (!attr && !h->has_labels) return fail(GK_ERR_ARG, "gk_pk_features: vertex labels are required");
  if (!attr && h->n_labels0 > dim) return fail(GK_ERR_ARG, "gk_pk_features: a label id is >= dim");
  const int64_t N = h->N, V = h->V, E = h->E, V1 = std::max<int64_t>(V, 1);
  const int K = attr ? dim : 1;
  const int64_t launches0 = h->launches;
  features_begin(h);
  h->pk_levels = 0;

  // the dense P the reference also holds on the host: refuse clearly when it cannot fit
  const size_t p_bytes = 2 * (size_t)V1 * dim * 8, bin_bytes = (size_t)t_max * V1 * K * 8;
  size_t free_b = 0, total_b = 0;
  GK_CUDA(cudaMemGetInfo(&free_b, &total_b));
  if (p_bytes + bin_bytes > free_b + h->pk_P.cap + h->pk_bins.cap)
    return fail(GK_ERR_RANGE, "gk_pk_features: the dense V x D propagation matrix (" + std::to_string(p_bytes >> 20) +
                                  " MiB double-buffered) and the bins (" + std::to_string(bin_bytes >> 20) +
                                  " MiB) do not fit in device memory");
  GK_TRY(h->pk_P.ensure(p_bytes));
  GK_TRY(h->pk_bins.ensure(bin_bytes));
  GK_TRY(h->pk_priv.ensure((size_t)t_max * V1));
  GK_TRY(h->pk_tval.ensure((size_t)std::max<int64_t>(E, 1) * 8));
  GK_TRY(h->pk_u.ensure((size_t)t_max * dim * 8));
  GK_TRY(h->pk_b.ensure((size_t)t_max * K * 8));
  GK_TRY(h->pk_cnt.ensure(24));  // [near-edge count u64 | NaN seen u32, pad | columns u64]
  double* P0 = h->pk_P.as<double>();
  double* P1 = P0 + (size_t)V1 * dim;
  double* bins = h->pk_bins.as<double>();
  unsigned char* priv = h->pk_priv.as<unsigned char>();
  unsigned long long* near = h->pk_cnt.as<unsigned long long>();
  unsigned* nan_seen = reinterpret_cast<unsigned*>(near + 1);
  GK_CUDA(cudaMemsetAsync(h->pk_cnt.p, 0, 24, h->stream));
  GK_CUDA(cudaMemsetAsync(priv, 0, (size_t)t_max * V1, h->stream));
  if (E) GK_CUDA(cudaMemcpyAsync(h->pk_tval.p, t_values, (size_t)E * 8, cudaMemcpyHostToDevice, h->stream));
  GK_CUDA(cudaMemcpyAsync(h->pk_u.p, u, (size_t)t_max * dim * 8, cudaMemcpyHostToDevice, h->stream));
  GK_CUDA(cudaMemcpyAsync(h->pk_b.p, b, (size_t)t_max * K * 8, cudaMemcpyHostToDevice, h->stream));
  if (attr) {
    if (V) GK_CUDA(cudaMemcpyAsync(P0, p0, (size_t)V * dim * 8, cudaMemcpyHostToDevice, h->stream));
  } else {
    GK_CUDA(cudaMemsetAsync(P0, 0, (size_t)V1 * dim * 8, h->stream));
    if (V) {
      pk_onehot<<<cdiv(V, 256), 256, 0, h->stream>>>((int)V, dim, h->labels0.as<int>(), P0);
      LAUNCH_CHECK(h);
    }
  }
  const int store = (flags & GK_PK_STORE_F32) ? PK_STORE_F32 : (flags & GK_PK_STORE_INT) ? PK_STORE_INT : PK_STORE_F64;
  const int v0 = h->graph_ptr_host[n_fit];  // first vertex of the transformed graphs

  // ---- levels: private flags, hash, propagate
  std::vector<cudaEvent_t> pev(2 * (size_t)t_max, nullptr);
  for (auto& e : pev) GK_CUDA(cudaEventCreate(&e));
  struct EvGuard {
    std::vector<cudaEvent_t>& v;
    ~EvGuard() { for (auto e : v) if (e) cudaEventDestroy(e); }
  } ev_guard{pev};
  GK_CUDA(cudaEventRecord(h->tev[2], h->stream));
  double* cur = P0;
  double* nxt = P1;
  const long long n_entries = (long long)V * dim;
  const int prop_grid = (int)std::max<long long>(1, std::min<long long>(cdiv(n_entries, 256), (long long)h->sm_count * 16));
  for (int t = 0; t < t_max && V; ++t) {
    if (split) {
      pk_private<<<cdiv(V, 256), 256, 0, h->stream>>>((int)V, v0, dim, dim_orig, t, h->labels0.as<int>(), cur,
                                                      priv + (size_t)t * V);
      LAUNCH_CHECK(h);
    }
    PkHashParams hp;
    hp.V = (int)V; hp.D = dim; hp.attr = attr ? 1 : 0; hp.take_sqrt = (flags & GK_PK_SQRT) ? 1 : 0;
    hp.dim_orig = dim_orig;
    hp.P = cur;
    hp.u = h->pk_u.as<double>() + (size_t)t * dim;
    hp.b = h->pk_b.as<double>() + (size_t)t * K;
    hp.w = w;
    hp.priv = split ? priv + (size_t)t * V : nullptr;
    hp.bins = bins + (size_t)t * V * K;
    hp.near = near; hp.nan_seen = nan_seen;
    pk_hash<<<cdiv(V, 256), 256, 0, h->stream>>>(hp);
    LAUNCH_CHECK(h);
    if (t + 1 < t_max) {
      GK_CUDA(cudaEventRecord(pev[2 * t], h->stream));
      pk_propagate<<<prop_grid, 256, 0, h->stream>>>(n_entries, dim, h->row_ptr.as<int>(), h->col_idx.as<int>(),
                                                     h->pk_tval.as<double>(), cur, nxt, store, near);
      LAUNCH_CHECK(h);
      GK_CUDA(cudaEventRecord(pev[2 * t + 1], h->stream));
      std::swap(cur, nxt);
    }
  }
  GK_CUDA(cudaEventRecord(h->tev[5], h->stream));

  // ---- per-level columns and (graph, column) counts
  const size_t cap = std::max<size_t>(next_pow2((size_t)V1 * 2), 1024);
  const size_t ft_cap = std::max<size_t>(next_pow2((size_t)t_max * (V1 + N) * 2), 1024);
  if (ft_cap > (1ULL << 31)) return fail(GK_ERR_ARG, "gk_pk_features: feature table too large");
  GK_TRY(h->pk_tab.ensure(cap * 8 + (size_t)V1 * 8));  // slot -> claiming vertex | slot -> column | vertex -> slot | ones
  int* tab = h->pk_tab.as<int>();
  int* colid = tab + cap;
  int* slot_of = colid + cap;
  unsigned char* ones = reinterpret_cast<unsigned char*>(slot_of + V1);
  GK_TRY(h->ft_keys.ensure(ft_cap * 8));
  GK_TRY(h->ft_cnt.ensure(ft_cap * 4));
  h->ft_cap = ft_cap;
  GK_TRY(init_scalars(h, 0));
  const int nbv = cdiv(V1, 256);
  FeatStats fst;
  GK_TRY(reset_feature_stats(h, (int64_t)t_max * V1, 2LL * t_max * nbv, &fst));
  GK_CUDA(cudaMemsetAsync(h->ft_keys.p, 0xFF, ft_cap * 8, h->stream));
  GK_CUDA(cudaMemsetAsync(h->ft_cnt.p, 0, ft_cap * 4, h->stream));
  GK_CUDA(cudaMemsetAsync(ones, 1, (size_t)V1, h->stream));
  unsigned long long* n_cols_d = near + 2;
  for (int t = 0; t < t_max && V; ++t) {
    const double* bt = bins + (size_t)t * V * K;
    const unsigned char* pt = split ? priv + (size_t)t * V : nullptr;
    GK_CUDA(cudaMemsetAsync(tab, 0xFF, cap * 4, h->stream));
    pk_code_insert<<<nbv, 256, 0, h->stream>>>((int)V, K, bt, pt, tab, (unsigned)(cap - 1), slot_of);
    LAUNCH_CHECK(h);
    nh_code_number<<<nbv, 256, 0, h->stream>>>((int)V, ones, tab, slot_of, colid, n_cols_d);
    LAUNCH_CHECK(h);
    pk_count<<<nbv, 256, 0, h->stream>>>((int)V, h->vgraph.as<int>(), h->graph_ptr.as<int>(), slot_of, colid,
                                         h->ft_keys.as<unsigned long long>(), h->ft_cnt.as<unsigned>(),
                                         (unsigned)(ft_cap - 1), fst, t, split ? 1 : 0, (int)n_fit,
                                         (size_t)t_max * nbv + (size_t)t * nbv);
    LAUNCH_CHECK(h);
  }
  GK_CUDA(cudaEventRecord(h->tev[3], h->stream));
  unsigned long long hc[3] = {0, 0, 0};
  GK_CUDA(cudaMemcpyAsync(hc, h->pk_cnt.p, 24, cudaMemcpyDeviceToHost, h->stream));
  DevScalars* hs;
  GK_TRY(read_scalars(h, &hs));  // synchronises
  if (hs->ft_overflow) return fail(GK_ERR_STATE, "gk_pk_features: feature table overflow");
  if ((unsigned)hc[1]) return fail(GK_ERR_UNSUPPORTED, "gk_pk_features: a bin is NaN (sqrt of a negative entry, or a NaN "
                                                       "input), which the reference cannot look up either");
  h->n_columns = (int64_t)hc[2];
  h->pk_levels = t_max;
  h->pk_K = K;
  features_publish(h, FK_PK);
  if (stats) {
    memset(stats, 0, sizeof(*stats));
    stats->n_graphs = N; stats->n_vertices = V; stats->n_edges = E;
    stats->n_levels = t_max;
    stats->n_columns = h->n_columns;
    stats->kernel_launches = h->launches - launches0;
    stats->ms_features = ev_ms(h->tev[2], h->tev[3]);
    stats->ms_hash = ev_ms(h->tev[2], h->tev[5]);
    stats->ms_columns = ev_ms(h->tev[5], h->tev[3]);
    float mp = 0.f;
    for (int t = 0; t + 1 < t_max && V; ++t) mp += ev_ms(pev[2 * t], pev[2 * t + 1]);
    stats->ms_propagate = mp;
    stats->pk_near_edge = (int64_t)hc[0];
  }
  return GK_OK;
}

int gk_pk_hashes(gk_handle* h, int32_t level, double* out, uint8_t* priv) {
  if (!h || !out) return fail(GK_ERR_ARG, "gk_pk_hashes: null argument");
  if (h->feature_kind != FK_PK || level < 0 || level >= h->pk_levels)
    return fail(GK_ERR_STATE, "gk_pk_hashes: no such level (run gk_pk_features first)");
  GK_CUDA(cudaSetDevice(h->dev));
  const size_t V = (size_t)h->V, K = (size_t)h->pk_K;
  if (V) {
    GK_CUDA(cudaMemcpyAsync(out, h->pk_bins.as<double>() + (size_t)level * V * K, V * K * 8, cudaMemcpyDeviceToHost,
                            h->stream));
    if (priv)
      GK_CUDA(cudaMemcpyAsync(priv, h->pk_priv.as<unsigned char>() + (size_t)level * V, V, cudaMemcpyDeviceToHost,
                              h->stream));
    GK_CUDA(cudaStreamSynchronize(h->stream));
  }
  return GK_OK;
}

// Launch rw_pairs over `n_pairs` pairs: the iteration vectors in shared memory when `vec_elems` doubles fit, else in
// a global workspace slice per CTA.  The workspace holds one slice per CTA of the clamped grid and at most 896 MiB of
// slices (1 GiB with DevBuf's growth slack): fewer CTAs, down to one, when a slice is large.
static int rw_launch(gk_handle* h, RwParams p, size_t vec_elems) {
  if (p.n_pairs <= 0) return GK_OK;
  const size_t bytes = vec_elems * 8;
  long long grid;
  size_t smem = 0;
  if (bytes <= RW_SMEM_MAX) {
    smem = bytes;
    GK_CUDA(cudaFuncSetAttribute(rw_pairs, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max<size_t>(smem, 1)));
    int per_sm = 0;
    GK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, rw_pairs, RW_THREADS, smem));
    grid = std::min<long long>((long long)h->sm_count * std::max(per_sm, 1), p.n_pairs);
    p.ws = nullptr;
  } else {
    grid = std::min<long long>((long long)h->sm_count * 2, p.n_pairs);
    grid = std::min(grid, std::max<long long>(1, (long long)((size_t)(896 << 20) / bytes)));
    GK_TRY(h->rw_ws.ensure((size_t)grid * bytes));
    p.ws = h->rw_ws.as<double>();
    p.ws_stride = (long long)vec_elems;
  }
  rw_pairs<<<(int)grid, RW_THREADS, smem, h->stream>>>(p);
  LAUNCH_CHECK(h);
  return GK_OK;
}

// Gram of the random walk kernels (gram_path 8 conjugate gradients, 9 spectral, 10 power series): fp64, host or
// GK_OUT_DEVICE output, GK_NORMALIZE, n_fit and row ranges.  Self similarities come from the same pair kernel, so a
// square K's diagonal equals them bit for bit.  The full square case computes the upper triangle and mirrors it.
static int gram_rw(gk_handle* h, const GramReq& q, gk_stats* stats) {
  const int64_t N = h->N, n_fit = q.n_fit, k_rows = q.k_rows, k_cols = q.k_cols;
  const bool square = q.square;
  const int64_t launches0 = h->launches;
  F64Out out;
  GK_TRY(f64_target(h, q, &out));
  GK_TRY(h->diag_f64.ensure((size_t)N * 8));
  GK_TRY(h->rw_iters.ensure((size_t)std::max<int64_t>(k_rows * k_cols, 1)));
  GK_CUDA(cudaMemsetAsync(h->rw_cap.p, 0, 8, h->stream));
  // largest vertex count among the row graphs and among the column graphs: the vectors of the largest pair
  auto max_n = [&](int64_t g0, int64_t g1) {
    int m = 0;
    for (int64_t g = g0; g < g1; ++g) m = std::max(m, h->graph_ptr_host[g + 1] - h->graph_ptr_host[g]);
    return (size_t)m;
  };
  const size_t nmax_all = max_n(0, N);
  const int nvec = h->rw_route == GK_RW_CG ? 3 : h->rw_route == GK_RW_SERIES ? 2 : 0;
  RwParams p;
  memset(&p, 0, sizeof(p));
  p.graph_ptr = h->graph_ptr.as<int>();
  p.row_ptr = h->row_ptr.as<int>(); p.col_idx = h->col_idx.as<int>(); p.val = h->rw_val.as<double>();
  p.trow_ptr = h->rw_trp.as<int>(); p.tcol_idx = h->rw_tci.as<int>(); p.tval = h->rw_tval.as<double>();
  p.labels = h->rw_labeled ? h->labels0.as<int>() : nullptr;
  p.q = h->rw_q.as<double>(); p.w = h->rw_w.as<double>();
  p.coef = h->rw_coef.as<double>(); p.n_coef = h->rw_ncoef;
  p.lamda = h->rw_lamda;
  p.route = h->rw_route; p.fn = h->rw_fn;
  p.cap_hits = h->rw_cap.as<unsigned long long>();
  GK_CUDA(cudaEventRecord(h->tev[2], h->stream));
  // self similarities of every graph
  {
    RwParams d = p;
    d.pairs = RW_PAIRS_DIAG;
    d.n_pairs = N;
    d.out = h->diag_f64.as<double>();
    GK_TRY(rw_launch(h, d, (size_t)nvec * nmax_all * nmax_all));
  }
  const bool mirror = q.full_square && !(q.flags & GK_FULL_TILES);
  if (k_rows > 0) {
    RwParams k = p;
    k.pairs = mirror ? RW_PAIRS_TRIANGLE : RW_PAIRS_RECT;
    k.ordered = square ? 1 : 0;
    k.n_pairs = mirror ? N * (N + 1) / 2 : k_rows * k_cols;
    k.row_g0 = q.a0;
    k.rows = (int)k_rows; k.cols = (int)k_cols;
    k.out = out.p; k.ld = out.ld;
    k.iters = h->rw_iters.as<unsigned char>();
    const size_t nr = mirror ? nmax_all : max_n(q.a0, q.a1), nc = max_n(0, n_fit);
    GK_TRY(rw_launch(h, k, (size_t)nvec * nr * nc));
  }
  h->rw_iter_rows = k_rows; h->rw_iter_cols = k_cols;
  GK_TRY(f64_deliver(h, q, out, true, h->tev[3], h->tev[4]));
  unsigned long long cap_hits = 0;
  GK_CUDA(cudaMemcpyAsync(&cap_hits, h->rw_cap.p, 8, cudaMemcpyDeviceToHost, h->stream));
  GK_CUDA(cudaStreamSynchronize(h->stream));
  if (stats) {
    stats->n_graphs = N; stats->n_vertices = h->V; stats->n_edges = h->E;
    stats->gram_path = h->rw_route == GK_RW_CG ? 8 : h->rw_route == GK_RW_SPECTRAL ? 9 : 10;
    stats->gemm_tiles = mirror ? N * (N + 1) / 2 : k_rows * k_cols;
    stats->gemm_launches = h->launches - launches0;
    stats->ms_rw = ev_ms(h->tev[2], h->tev[3]);
    stats->ms_gemm = stats->ms_rw;
    stats->ms_d2h = ev_ms(h->tev[3], h->tev[4]);
    stats->ms_total = stats->ms_rw + stats->ms_d2h;
    stats->rw_cap_hits = (int64_t)cap_hits;
  }
  return GK_OK;
}

// ---------------------------------------------------------------------------
// SubgraphMatching (subgraph_matching.cuh).  gk_sm_features builds every graph's record and uploads the weight
// tables and lambdas; gk_gram (gram_sm) runs one warp per graph pair.
static bool sm_integral(const double* t, int64_t n) {
  for (int64_t i = 0; i < n; ++i)
    if (t[i] != std::floor(t[i])) return false;
  return true;
}

// gk_sm_features without the publication: the relabelling frameworks publish after adding their levels
static int sm_features_impl(gk_handle* h, int32_t k, const double* lambdas, const double* vtable, int32_t n_vlabels,
                            const double* etable, int32_t n_elabels, const int32_t* edge_label, int32_t flags,
                            gk_stats* stats) {
  GK_TRY(need_packed(h, "gk_sm_features"));
  if (flags & ~(GK_SM_KV_NONE | GK_SM_KV_DIRAC | GK_SM_KE_NONE | GK_SM_KE_DIRAC))
    return fail(GK_ERR_ARG, "gk_sm_features: unknown flags");
  if ((flags & GK_SM_KV_NONE) && (flags & GK_SM_KV_DIRAC)) return fail(GK_ERR_ARG, "gk_sm_features: two vertex kernels");
  if ((flags & GK_SM_KE_NONE) && (flags & GK_SM_KE_DIRAC)) return fail(GK_ERR_ARG, "gk_sm_features: two edge kernels");
  if (k < 0 || !lambdas) return fail(GK_ERR_ARG, "gk_sm_features: k < 0 or no lambdas");
  const int kv = (flags & GK_SM_KV_NONE) ? SM_W_NONE : (flags & GK_SM_KV_DIRAC) ? SM_W_DIRAC : SM_W_TABLE;
  const int ke = (flags & GK_SM_KE_NONE) ? SM_W_NONE : (flags & GK_SM_KE_DIRAC) ? SM_W_DIRAC : SM_W_TABLE;
  if (kv != SM_W_NONE && !h->has_labels) return fail(GK_ERR_ARG, "gk_sm_features: the vertex kernel needs packed labels");
  if (ke != SM_W_NONE && h->E > 0 && !edge_label) return fail(GK_ERR_ARG, "gk_sm_features: the edge kernel needs edge labels");
  const int64_t nvt = (int64_t)n_vlabels * n_vlabels, net = (int64_t)n_elabels * n_elabels;
  if (kv == SM_W_TABLE && (!vtable || n_vlabels < 1)) return fail(GK_ERR_ARG, "gk_sm_features: no vertex table");
  if (ke == SM_W_TABLE && (!etable || n_elabels < 1)) return fail(GK_ERR_ARG, "gk_sm_features: no edge table");
  if ((kv == SM_W_TABLE && nvt > SM_TAB_MAX) || (ke == SM_W_TABLE && net > SM_TAB_MAX))
    return fail(GK_ERR_UNSUPPORTED, "gk_sm_features: a weight table has more than 4096 entries (64 labels)");
  for (int64_t i = 0; kv == SM_W_TABLE && i < nvt; ++i)
    if (!std::isfinite(vtable[i])) return fail(GK_ERR_UNSUPPORTED, "gk_sm_features: non-finite vertex weight");
  for (int64_t i = 0; ke == SM_W_TABLE && i < net; ++i)
    if (!std::isfinite(etable[i])) return fail(GK_ERR_UNSUPPORTED, "gk_sm_features: non-finite edge weight");
  const int n_tv = k + 1;
  for (int i = 0; i < n_tv; ++i)
    if (!std::isfinite(lambdas[i])) return fail(GK_ERR_UNSUPPORTED, "gk_sm_features: non-finite lambda");
  if (n_tv > 15 && !sm_integral(lambdas, n_tv))
    return fail(GK_ERR_UNSUPPORTED, "gk_sm_features: real lambdas are folded in the reference's order for k + 1 <= 15 only");
  // cliques of the product graph have at most min(n_x, n_y) vertices
  const int kk = std::max(1, std::min(std::max(k, 1), h->max_graph_size));
  if (kk > SM_KMAX) return fail(GK_ERR_UNSUPPORTED, "gk_sm_features: subgraphs of more than 32 vertices");
  features_begin(h);
  h->sm_n_lv = 0;
  h->sm_hc = false;
  const int64_t N = h->N;
  const bool elab = ke != SM_W_NONE;
  std::vector<long long> off(N + 1, 0);
  for (int64_t g = 0; g < N; ++g) off[g + 1] = off[g] + sm_record_words(h->graph_ptr_host[g + 1] - h->graph_ptr_host[g], elab);
  GK_CUDA(cudaEventRecord(h->tev[0], h->stream));
  GK_TRY(h->sm_off.ensure((N + 1) * 8));
  GK_TRY(h->sm_rec.ensure(std::max<long long>(off[N], 1) * 4));
  GK_CUDA(cudaMemcpyAsync(h->sm_off.p, off.data(), (N + 1) * 8, cudaMemcpyHostToDevice, h->stream));
  GK_TRY(h->sm_el.ensure(std::max<int64_t>(h->E, 1) * 4));
  GK_TRY(h->sm_ctl.ensure(16));
  GK_CUDA(cudaMemsetAsync(h->sm_ctl.p, 0, 16, h->stream));
  int* d_max_und = reinterpret_cast<int*>(h->sm_ctl.as<unsigned char>() + 12);
  if (elab && h->E > 0) GK_CUDA(cudaMemcpyAsync(h->sm_el.p, edge_label, h->E * 4, cudaMemcpyHostToDevice, h->stream));
  sm_build_records<<<(int)std::min<int64_t>(N, h->sm_count * 16), 256, 0, h->stream>>>(
      h->graph_ptr.as<int>(), h->row_ptr.as<int>(), h->col_idx.as<int>(), kv != SM_W_NONE ? h->labels0.as<int>() : nullptr,
      elab ? h->sm_el.as<int>() : nullptr, h->sm_off.as<long long>(), h->sm_rec.as<unsigned>(), (int)N, d_max_und);
  LAUNCH_CHECK(h);
  GK_TRY(h->sm_vtab.ensure(std::max<int64_t>(nvt, 1) * 8));
  GK_TRY(h->sm_etab.ensure(std::max<int64_t>(net, 1) * 8));
  GK_TRY(h->sm_lam.ensure((size_t)n_tv * 8));
  if (kv == SM_W_TABLE) GK_CUDA(cudaMemcpyAsync(h->sm_vtab.p, vtable, nvt * 8, cudaMemcpyHostToDevice, h->stream));
  if (ke == SM_W_TABLE) GK_CUDA(cudaMemcpyAsync(h->sm_etab.p, etable, net * 8, cudaMemcpyHostToDevice, h->stream));
  GK_CUDA(cudaMemcpyAsync(h->sm_lam.p, lambdas, (size_t)n_tv * 8, cudaMemcpyHostToDevice, h->stream));
  int max_und = 0;
  GK_CUDA(cudaMemcpyAsync(&max_und, d_max_und, 4, cudaMemcpyDeviceToHost, h->stream));
  GK_CUDA(cudaEventRecord(h->tev[1], h->stream));
  GK_CUDA(cudaStreamSynchronize(h->stream));  // the caller's buffers may be reused once we return
  h->sm_max_und = max_und;
  h->sm_k = k; h->sm_kk = kk; h->sm_kv = kv; h->sm_ke = ke;
  h->sm_n_vl = kv == SM_W_TABLE ? n_vlabels : 0;
  h->sm_n_el = ke == SM_W_TABLE ? n_elabels : 0;
  h->sm_exact = (kv != SM_W_TABLE || sm_integral(vtable, nvt)) && (ke != SM_W_TABLE || sm_integral(etable, net));
  if (stats) {
    stats->n_graphs = N; stats->n_vertices = h->V; stats->n_edges = h->E;
    stats->ms_h2d = ev_ms(h->tev[0], h->tev[1]);
  }
  return GK_OK;
}

int gk_sm_features(gk_handle* h, int32_t k, const double* lambdas, const double* vtable, int32_t n_vlabels,
                   const double* etable, int32_t n_elabels, const int32_t* edge_label, int32_t flags, gk_stats* stats) {
  GK_TRY(sm_features_impl(h, k, lambdas, vtable, n_vlabels, etable, n_elabels, edge_label, flags, stats));
  features_publish(h, FK_SM);
  return GK_OK;
}

// Launch sm_pairs over p.n_pairs pairs: a persistent grid, each warp with a stack slice sized for the deepest
// extension sets of the block and, when the two records of the largest pair fit, a shared-memory staging area.
static int sm_launch(gk_handle* h, SmParams p) {
  if (p.n_pairs <= 0) return GK_OK;
  const int nmax = std::max(h->max_graph_size, 1);
  const long long nv = (long long)nmax * nmax;
  // the extension set of S (|S| = d) lies in the c-neighbourhood of S: at most d D^2 vertices, D the largest number
  // of distinct out- or in-neighbours of a vertex (counted by sm_build_records)
  const long long D = h->sm_max_und;
  long long cap = 1;
  for (int d = 1; d < p.kk; ++d) cap += std::min(nv, d * D * D);
  p.stack_cap = cap;
  const size_t tab_bytes = ((p.kv == SM_W_TABLE ? (size_t)p.n_vl * p.n_vl : 0) +
                            (p.ke == SM_W_TABLE ? (size_t)p.n_el * p.n_el : 0)) * 8;
  // sm_wl_pairs' (depth, size) and sm_mask_pairs' (level, size) bins: per warp when exact, per lane when real
  const size_t bin_bytes = p.n_lv == 0 ? 0 : (size_t)p.n_lv * p.kk * 8 * (p.exact ? 2 * SM_WARPS : SM_THREADS);
  const long long pair_words = 2 * sm_record_words(nmax, p.ke != SM_W_NONE);
  // GRAKEL_B200_SM_GLOBAL=1 reads every record from global memory (the route of pairs too large to stage)
  const char* e_glob = getenv("GRAKEL_B200_SM_GLOBAL");
  const bool staged =
      !(e_glob && atoi(e_glob) != 0) && tab_bytes + bin_bytes + SM_WARPS * pair_words * 4 <= 96 * 1024;
  p.stage_words = staged ? (int)pair_words : 0;
  const size_t smem = tab_bytes + bin_bytes + (size_t)SM_WARPS * p.stage_words * 4;
  const void* kern = p.n_lv == 0 ? (const void*)sm_pairs : h->sm_hc ? (const void*)sm_mask_pairs : (const void*)sm_wl_pairs;
  GK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max<size_t>(smem, 1)));
  int per_sm = 0;
  GK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, SM_THREADS, smem));
  long long grid = (long long)h->sm_count * std::max(per_sm, 1);
  // at most 1 GiB of stacks: fewer CTAs (down to one) when a lane's stack is large
  const long long per_cta = (long long)SM_WARPS * 32 * cap * 4;
  grid = std::min(grid, std::max<long long>(1, (1LL << 30) / per_cta));
  grid = std::min<long long>(grid, (p.n_pairs + SM_WARPS - 1) / SM_WARPS);
  GK_TRY(h->sm_stack.ensure((size_t)grid * per_cta));
  p.stack = h->sm_stack.as<unsigned>();
  GK_CUDA(cudaMemsetAsync(h->sm_ctl.p, 0, 8, h->stream));
  p.next = h->sm_ctl.as<unsigned long long>();
  if (p.n_lv > 0 && h->sm_hc)
    sm_mask_pairs<<<(int)grid, SM_THREADS, smem, h->stream>>>(p);
  else if (p.n_lv > 0)
    sm_wl_pairs<<<(int)grid, SM_THREADS, smem, h->stream>>>(p);
  else
    sm_pairs<<<(int)grid, SM_THREADS, smem, h->stream>>>(p);
  LAUNCH_CHECK(h);
  return GK_OK;
}

static SmParams sm_params(gk_handle* h) {
  SmParams p;
  memset(&p, 0, sizeof(p));
  p.graph_ptr = h->graph_ptr.as<int>();
  p.rec_off = h->sm_off.as<long long>(); p.rec = h->sm_rec.as<unsigned>();
  p.vtab = h->sm_vtab.as<double>(); p.n_vl = h->sm_n_vl;
  p.etab = h->sm_etab.as<double>(); p.n_el = h->sm_n_el;
  p.kv = h->sm_kv; p.ke = h->sm_ke;
  p.kk = h->sm_kk; p.n_tv = h->sm_k + 1;
  p.lam = h->sm_lam.as<double>();
  p.exact = h->sm_exact ? 1 : 0;
  p.err = reinterpret_cast<unsigned*>(h->sm_ctl.as<unsigned char>() + 8);
  p.wl_cls = h->sm_wl_cls.as<int>(); p.n_lv = h->sm_n_lv;
  return p;
}

static int sm_check_err(gk_handle* h) {
  unsigned err = 0;
  GK_CUDA(cudaMemcpyAsync(&err, h->sm_ctl.as<unsigned char>() + 8, 4, cudaMemcpyDeviceToHost, h->stream));
  GK_CUDA(cudaStreamSynchronize(h->stream));
  if (err & 1u) return fail(GK_ERR_RANGE, "SubgraphMatching: a clique count reached 2^53, past exact fp64");
  if (err & 2u) return fail(GK_ERR_RANGE, "SubgraphMatching: an extension set overflowed its stack");
  return GK_OK;
}

// Gram of SubgraphMatching (gram_path 13): fp64, host or GK_OUT_DEVICE output, GK_NORMALIZE, n_fit and row ranges.
// The self similarities come from the same pair kernel, so a square K's diagonal equals them bit for bit; the full
// square case computes the upper triangle and mirrors it.
static int gram_sm(gk_handle* h, const GramReq& q, gk_stats* stats) {
  const int64_t N = h->N, k_rows = q.k_rows, k_cols = q.k_cols;
  const int64_t launches0 = h->launches;
  F64Out out;
  GK_TRY(f64_target(h, q, &out));
  GK_TRY(h->diag_f64.ensure((size_t)N * 8));
  GK_CUDA(cudaMemsetAsync(h->sm_ctl.as<unsigned char>() + 8, 0, 8, h->stream));
  const SmParams p = sm_params(h);
  GK_CUDA(cudaEventRecord(h->tev[2], h->stream));
  {
    SmParams d = p;
    d.pairs = RW_PAIRS_DIAG;
    d.n_pairs = N;
    d.out = h->diag_f64.as<double>();
    GK_TRY(sm_launch(h, d));
  }
  const bool mirror = q.full_square && !(q.flags & GK_FULL_TILES);
  if (k_rows > 0) {
    SmParams k = p;
    k.pairs = mirror ? RW_PAIRS_TRIANGLE : RW_PAIRS_RECT;
    k.ordered = q.square ? 1 : 0;
    k.n_pairs = mirror ? N * (N + 1) / 2 : k_rows * k_cols;
    k.row_g0 = q.a0;
    k.rows = (int)k_rows; k.cols = (int)k_cols;
    k.out = out.p; k.ld = out.ld;
    GK_TRY(sm_launch(h, k));
  }
  GK_CUDA(cudaEventRecord(h->tev[3], h->stream));
  GK_TRY(sm_check_err(h));
  GK_TRY(f64_deliver(h, q, out, true, h->tev[3], h->tev[4]));
  if (stats) {
    stats->n_graphs = N; stats->n_vertices = h->V; stats->n_edges = h->E;
    stats->gram_path = 13;
    stats->gemm_tiles = mirror ? N * (N + 1) / 2 : k_rows * k_cols;
    stats->gemm_launches = h->launches - launches0;
    stats->ms_rw = ev_ms(h->tev[2], h->tev[3]);
    stats->ms_gemm = stats->ms_rw;
    stats->ms_d2h = ev_ms(h->tev[3], h->tev[4]);
    stats->ms_total = stats->ms_rw + stats->ms_d2h;
  }
  return GK_OK;
}

// tv of every level of the n_fit pairs of row `row`: out[n_fit][n_lv][k + 1] (gk_sm_wl_features' levels) or
// out[n_fit][k + 1]
static int sm_counts(gk_handle* h, int64_t n_fit, int64_t row, double* out, const char* what) {
  if (n_fit <= 0 || n_fit > h->N) return fail(GK_ERR_ARG, std::string(what) + ": n_fit out of range");
  const bool square = n_fit == h->N;
  if (row < 0 || row >= (square ? h->N : h->N - n_fit)) return fail(GK_ERR_ARG, std::string(what) + ": row out of range");
  GK_CUDA(cudaSetDevice(h->dev));
  const size_t bytes = (size_t)n_fit * std::max(h->sm_n_lv, 1) * (h->sm_k + 1) * 8;
  GK_TRY(h->K_stage.ensure(bytes));
  GK_CUDA(cudaMemsetAsync(h->sm_ctl.as<unsigned char>() + 8, 0, 8, h->stream));
  SmParams p = sm_params(h);
  p.pairs = RW_PAIRS_RECT;
  p.ordered = square ? 1 : 0;
  p.n_pairs = n_fit;
  p.row_g0 = (int)((square ? 0 : n_fit) + row);
  p.rows = 1; p.cols = (int)n_fit;
  p.tv_out = h->K_stage.as<double>();
  GK_TRY(sm_launch(h, p));
  GK_TRY(sm_check_err(h));
  GK_CUDA(cudaMemcpyAsync(out, h->K_stage.p, bytes, cudaMemcpyDeviceToHost, h->stream));
  GK_CUDA(cudaStreamSynchronize(h->stream));
  return GK_OK;
}

int gk_sm_counts(gk_handle* h, int64_t n_fit, int64_t row, double* out) {
  if (!h || !out) return fail(GK_ERR_ARG, "gk_sm_counts: null argument");
  if (h->feature_kind != FK_SM || h->sm_n_lv != 0)
    return fail(GK_ERR_STATE, "gk_sm_counts: call gk_sm_features first");
  return sm_counts(h, n_fit, row, out, "gk_sm_counts");
}


// A relabelling framework over SubgraphMatching: gk_sm_features' records, tables and lambdas, and the class of every
// packed vertex at each of n_lv levels; gk_gram then returns the level sum of the per-level SubgraphMatching Grams from
// one enumeration per pair.  Levels that refine each other (WL) run sm_wl_pairs, others (HadamardCode) sm_mask_pairs.
static int sm_level_features(gk_handle* h, const char* fn, int32_t k, int32_t n_iter, int n_lv, int bins,
                             const char* cap_msg, bool refine, const int32_t* level_ids, const double* lambdas,
                             const double* etable, int32_t n_elabels, const int32_t* edge_label, int32_t flags,
                             gk_stats* stats) {
  GK_TRY(need_packed(h, fn));
  if (n_iter < 1) return fail(GK_ERR_ARG, std::string(fn) + ": n_iter < 1");
  if (!(flags & (GK_SM_KV_NONE | GK_SM_KV_DIRAC)))
    return fail(GK_ERR_UNSUPPORTED, std::string(fn) + ": the vertex kernel must be GK_SM_KV_DIRAC or GK_SM_KV_NONE");
  const bool all_levels = (flags & GK_SM_KV_NONE) != 0;
  if (!all_levels && !level_ids) return fail(GK_ERR_ARG, std::string(fn) + ": no level ids");
  const int kk = std::max(1, std::min(std::max(k, 1), h->max_graph_size));
  if ((int64_t)n_lv * kk > bins) return fail(GK_ERR_UNSUPPORTED, std::string(fn) + ": " + cap_msg);
  GK_TRY(sm_features_impl(h, k, lambdas, nullptr, 0, etable, n_elabels, edge_label, flags, stats));
  const size_t bytes = (size_t)h->V * n_lv * 4;
  GK_TRY(h->sm_wl_cls.ensure(std::max<size_t>(bytes, 4)));
  if (!all_levels && bytes > 0) {
    GK_CUDA(cudaMemcpyAsync(h->sm_wl_cls.p, level_ids, bytes, cudaMemcpyHostToDevice, h->stream));
    GK_CUDA(cudaStreamSynchronize(h->stream));  // the caller's buffer may be reused once we return
  }
  h->sm_n_lv = n_lv;
  h->sm_hc = !refine;
  features_publish(h, FK_SM);
  return GK_OK;
}

// WeisfeilerLehman over SubgraphMatching (sm_wl_pairs): the WL class of every packed vertex at every level 0 .. n_iter
int gk_sm_wl_features(gk_handle* h, int32_t k, int32_t n_iter, const int32_t* level_ids, const double* lambdas,
                      const double* etable, int32_t n_elabels, const int32_t* edge_label, int32_t flags,
                      gk_stats* stats) {
  return sm_level_features(h, "gk_sm_wl_features", k, n_iter, n_iter + 1, SM_WL_BINS,
                           "(n_iter + 1) * min(k, largest graph) is more than 64", true, level_ids, lambdas, etable,
                           n_elabels, edge_label, flags, stats);
}

int gk_sm_wl_counts(gk_handle* h, int64_t n_fit, int64_t row, double* out) {
  if (!h || !out) return fail(GK_ERR_ARG, "gk_sm_wl_counts: null argument");
  if (h->feature_kind != FK_SM || h->sm_n_lv == 0 || h->sm_hc)
    return fail(GK_ERR_STATE, "gk_sm_wl_counts: call gk_sm_wl_features first");
  return sm_counts(h, n_fit, row, out, "gk_sm_wl_counts");
}

// HadamardCode over SubgraphMatching (sm_mask_pairs): the HadamardCode class of every packed vertex at every level
// 0 .. n_iter - 1
int gk_sm_hc_features(gk_handle* h, int32_t k, int32_t n_iter, const int32_t* level_ids, const double* lambdas,
                      const double* etable, int32_t n_elabels, const int32_t* edge_label, int32_t flags,
                      gk_stats* stats) {
  return sm_level_features(h, "gk_sm_hc_features", k, n_iter, n_iter, SM_HC_BINS,
                           "n_iter * min(k, largest graph) is more than 64", false, level_ids, lambdas, etable,
                           n_elabels, edge_label, flags, stats);
}

// ---------------------------------------------------------------------------
}  // extern "C"

// ---------------------------------------------------------------------------
// Host delivery of an fp32 device matrix into the caller's float64 array (host_deliver.h): K is moved as
// fp32 -- for the symmetric square case only its upper triangle, in row bands of roughly equal area --
// through a ring of pinned staging buffers; host threads widen each band into the destination rows and
// write the mirrored half (8 x 8 register transposes) while the next bands are on the PCIe bus.
#include "host_deliver.h"

// Symmetric integer-valued fp32 result -> the caller's float64 host matrix: upper triangle over PCIe in the narrowest
// exact type (u16 when the largest self similarity is below 2^16, packed band by band on the device first; else fp32),
// widened and mirrored by the host pool (host_deliver.h).
static int deliver_square(gk_handle* h, const float* d_k, long long d_ld, int64_t k_rows, double* dst, int64_t ld, int64_t max_diag) {
  DeviceCopier cp{h};
  if (max_diag < 65536 && !getenv("GRAKEL_B200_NO_U16")) {
    const std::vector<long long> start = tri_bands(k_rows);
    const int nb = (int)start.size() - 1;
    std::vector<long long> tab(start);
    long long off = 0;
    for (int c = 0; c < nb; ++c) { tab.push_back(off); off += (start[c + 1] - start[c]) * (k_rows - start[c]); }
    GK_TRY(h->K_stage.ensure((size_t)off * 2 + tab.size() * 8 + 64));
    GK_TRY(h->h_bands.ensure(tab.size() * 8));
    memcpy(h->h_bands.p, tab.data(), tab.size() * 8);
    long long* d_tab = reinterpret_cast<long long*>(h->K_stage.as<char>() + (((size_t)off * 2 + 63) / 64 * 64));
    GK_CUDA(cudaMemcpyAsync(d_tab, h->h_bands.p, tab.size() * 8, cudaMemcpyHostToDevice, h->stream));
    pack_tri_u16<<<h->sm_count * 8, 256, 0, h->stream>>>(d_k, d_ld, k_rows, d_tab, d_tab + nb + 1, nb, h->K_stage.as<unsigned short>());
    LAUNCH_CHECK(h);
    return deliver_tri<uint16_t>(cp, h->K_stage.as<uint16_t>(), 0, k_rows, dst, ld);
  }
  return deliver_tri<float>(cp, d_k, d_ld, k_rows, dst, ld);
}

template <typename OutT, bool NORM>
static void launch_tc(gk_handle* h, const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmC,
                      const GramParams& p, int grid, int elem_bytes) {
  if (elem_bytes == 1) gram_tc_kernel<OutT, NORM, 2><<<grid, GEMM_THREADS, GEMM_SMEM, h->stream>>>(tmA, tmB, tmC, p);
  else gram_tc_kernel<OutT, NORM, 0><<<grid, GEMM_THREADS, GEMM_SMEM, h->stream>>>(tmA, tmB, tmC, p);
}
template <typename OutT, bool NORM>
static void launch_simt(gk_handle* h, const unsigned* panel, long long ldp, int kdim, int a0, int a1, int b0, int b1,
                        const GramParams& p) {
  dim3 grid(cdiv(b1 - b0, 16), cdiv(a1 - a0, 16));
  gram_simt_kernel<OutT, NORM><<<grid, 256, 0, h->stream>>>(panel, ldp, kdim, a0, a1, b0, b1, p);
}
template <typename OutT, bool NORM>
static void launch_empty(gk_handle* h, int a0, int a1, int b0, int b1, const GramParams& p) {
  gram_empty_kernel<OutT, NORM><<<h->sm_count * 4, 256, 0, h->stream>>>(a0, a1, b0, b1, p);
}

// Build the tile list: bands of 12 row tiles, column-major inside a band, so that the
// ~132 tiles in flight (one per SM) cover a compact block of the output and share panel rows in L2.
static void build_tiles(std::vector<int2>& tiles, int a0, int a1, int b0, int b1, bool upper_only, int bm) {
  const int n_m = cdiv(a1 - a0, bm), n_n = cdiv(b1 - b0, BN);
  const int BAND = 12 * BM / bm;
  for (int m0 = 0; m0 < n_m; m0 += BAND) {
    const int m1 = std::min(n_m, m0 + BAND);
    for (int j = 0; j < n_n; ++j) {
      for (int i = m0; i < m1; ++i) {
        const int ar = a0 + i * bm, br = b0 + j * BN;
        if (upper_only && br + BN - 1 < ar) continue;  // tile entirely below the diagonal
        tiles.push_back(make_int2(ar, br));
      }
    }
  }
}

// ---- multi-GPU helpers (collective: every rank of the communicator calls them in the same order)
static int comm_barrier(gk_handle* h) {
  Comm* c = reinterpret_cast<Comm*>(h->comm);
  NcclApi* api = nccl_api();
  GK_NCCL(api, api->AllReduce(c->d_token, c->d_token, 1, ncclInt32, ncclSum, c->comm, h->stream));
  return GK_OK;
}

// Make h->K (>= bytes, the same request on every rank) visible to the peers: CUDA IPC handles travel through one
// ncclAllGather; mappings are renewed only when the buffer had to grow (the same call on every rank).
static int comm_share_K(gk_handle* h, size_t bytes) {
  Comm* c = reinterpret_cast<Comm*>(h->comm);
  NcclApi* api = nccl_api();
  if (c->exported && c->exported == h->K.p && h->K.cap >= bytes) return GK_OK;
  // peers unmap the old buffer before anybody frees it
  for (int r = 0; r < c->nranks; ++r)
    if (r != c->rank && c->peer_base[r]) { cudaIpcCloseMemHandle(c->peer_base[r]); c->peer_base[r] = nullptr; }
  GK_TRY(comm_barrier(h));
  GK_CUDA(cudaStreamSynchronize(h->stream));
  GK_TRY(h->K.ensure(bytes));
  cudaIpcMemHandle_t mine;
  GK_CUDA(cudaIpcGetMemHandle(&mine, h->K.p));
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle is 64 bytes");
  unsigned char* d_mine = c->d_handles + (size_t)c->nranks * 64;
  GK_CUDA(cudaMemcpyAsync(d_mine, &mine, 64, cudaMemcpyHostToDevice, h->stream));
  GK_NCCL(api, api->AllGather(d_mine, c->d_handles, 64, ncclChar, c->comm, h->stream));
  std::vector<cudaIpcMemHandle_t> all(c->nranks);
  GK_CUDA(cudaMemcpyAsync(all.data(), c->d_handles, (size_t)c->nranks * 64, cudaMemcpyDeviceToHost, h->stream));
  GK_CUDA(cudaStreamSynchronize(h->stream));
  for (int r = 0; r < c->nranks; ++r) {
    if (r == c->rank) { c->peer_base[r] = h->K.p; continue; }
    GK_CUDA(cudaIpcOpenMemHandle(&c->peer_base[r], all[r], cudaIpcMemLazyEnablePeerAccess));
  }
  c->exported = h->K.p;
  c->exported_cap = h->K.cap;
  return GK_OK;
}

// The integer Gram of the counts in `fb` (gram_path 1 tensor cores, 2 CUDA cores, 3 no shared column), with the
// head/tail split of its columns, fp32 or fp64 output, GK_NORMALIZE, a row map and GK_DIST.
static int gram_int(gk_handle* h, const GramReq& q, const IntBlock& fb, gk_stats* stats) {
  const int64_t N = q.N, n_fit = q.n_fit, k_rows = q.k_rows, k_cols = q.k_cols, row_begin = q.row_begin, row_end = q.row_end;
  const int32_t flags = q.flags, out_dtype = q.out_dtype;
  const bool square = q.square;
  const int* d_row_map = q.row_map;
  const int64_t launches0 = h->launches;
  const bool normalize = flags & GK_NORMALIZE;
  const size_t esz = out_dtype == GK_F64 ? 8 : 4;
  DevScalars* sc = h->scalars.as<DevScalars>();

  GK_CUDA(cudaEventRecord(h->tev[4], h->stream));
  // ---- column statistics were maintained by the feature kernels; finish the self similarities
  const int64_t D = std::max<int64_t>(fb.n_columns, 1);
  if (D > fb.col_cap) return fail(GK_ERR_STATE, "gk_gram: column statistics missing");
  const int nbc = cdiv(D, 256);
  GK_TRY(h->colslot.ensure(D * 4));
  GK_TRY(h->colstats.ensure(sizeof(ColStats)));
  GK_TRY(h->h_colstats.ensure(sizeof(ColStats)));
  GK_TRY(h->diag_f64.ensure(N * 8));
  const bool pro = square && !d_row_map && fb.prologue_on_host && D <= fb.col_cap;
  if (!pro) GK_CUDA(cudaMemsetAsync(&sc->n_entries, 0, sizeof(unsigned long long) * 3 + sizeof(long long), h->stream));
  const unsigned long long* d_diag_u64 = fb.diag;
  if (d_row_map) {
    GK_TRY(h->diag_rows.ensure(N * 8));
    GK_CUDA(cudaMemsetAsync(h->diag_rows.p, 0, N * 8, h->stream));
    diag_remap<<<cdiv(h->N, 256), 256, 0, h->stream>>>((int)h->N, d_row_map, d_diag_u64, h->diag_rows.as<unsigned long long>());
    LAUNCH_CHECK(h);
    d_diag_u64 = h->diag_rows.as<unsigned long long>();
  }
  if (!pro) {
    diag_finish<<<cdiv(N, 256), 256, 0, h->stream>>>((int)N, d_diag_u64,
                                                     h->diag_f64.as<double>(), (int)fb.n_part, fb.part_max,
                                                     fb.part_new, sc);
    LAUNCH_CHECK(h);
  }
  if (!square) {  // which columns occur on both the X and the Y side
    GK_TRY(h->colmin.ensure(D * 4));
    GK_TRY(h->colmax.ensure(D * 4));
    GK_CUDA(cudaMemsetAsync(h->colmin.p, 0x7F, D * 4, h->stream));
    GK_CUDA(cudaMemsetAsync(h->colmax.p, 0xFF, D * 4, h->stream));
    feat_minmax<<<h->sm_count * 16, 256, 0, h->stream>>>(fb.cap, fb.keys, d_row_map,
                                                         h->colmin.as<int>(), h->colmax.as<int>());
    LAUNCH_CHECK(h);
  }

  // ---- head / tail split.  force_T: 1 = every contributing column dense.
  const double flops_per_col = square ? (double)k_rows * (double)(N + 1) : 2.0 * (double)k_rows * (double)k_cols;
  const double store_seconds = (double)k_rows * (double)k_cols * (double)esz / 6.5e12;  // K written once (debug print only)
  int force_T = (flags & (GK_GRAM_SIMT | GK_DENSE_ALL)) ? 1 : -1;
  if (force_T < 0) {  // testing knob: GRAKEL_B200_FORCE_T=<threshold>
    const char* e = getenv("GRAKEL_B200_FORCE_T");
    if (e && *e) force_T = std::max(1, atoi(e));
  }
  ColStats* cs = h->colstats.as<ColStats>();
  ColStats hc;
  DevScalars* hs = nullptr;
  int64_t max_count, max_diag, n_entries;
  if (pro) {  // gk_wl_features ran diag_finish + col_hist and brought the results back with its own synchronisation
    hc = h->pro_hist;
    max_count = h->pro_max_count; max_diag = h->pro_max_diag; n_entries = h->pro_n_entries;
  } else {
    GK_CUDA(cudaMemsetAsync(cs, 0, sizeof(ColStats), h->stream));
    col_hist<<<nbc, 256, 0, h->stream>>>(D, square ? 1 : 0, (int)n_fit, fb.colcnt, h->colmin.as<int>(),
                                         h->colmax.as<int>(), cs);
    LAUNCH_CHECK(h);
    GK_CUDA(cudaMemcpyAsync(h->h_colstats.p, cs, sizeof(ColStats), cudaMemcpyDeviceToHost, h->stream));
    GK_TRY(read_scalars(h, &hs));  // the one host synchronisation of gk_gram
    hc = *h->h_colstats.as<ColStats>();
    max_count = (int64_t)hs->max_count; max_diag = (int64_t)hs->max_diag; n_entries = (int64_t)hs->n_entries;
  }
  // ---- choose the Gram path and the head/tail threshold (host side, from the histogram)
  int path = 1;
  if ((flags & GK_GRAM_SIMT) || max_count > 256 || max_diag >= (1LL << 24)) { path = 2; force_T = 1; }
  // panel element bytes of the tensor-core GEMM: u8 when every count fits, bf16 for a count of 256
  const int elem_bytes = (u8_panel_enabled() && max_count <= 255) ? 1 : 2;
  const int bk = panel_bk(elem_bytes);
  h->last_max_count = max_count;
  int T = 1;
  {
    // T = 2^k minimising  head_cols * flops_per_col / rate + tail_updates * t_atomic  (COST_GEMM_RATE_*, COST_T_ATOMIC)
    const double rate = panel_rate(elem_bytes);
    const double t_atomic = COST_T_ATOMIC;
    double best = -1.0;
    for (int k = 0; k <= HIST_BUCKETS - 2; ++k) {
      double head_cols = 0, tail_upd = 0;
      for (int b = 0; b < HIST_BUCKETS; ++b) {
        if (b > k) head_cols += (double)hc.hist_cols[b];
        else tail_upd += (double)hc.hist_work[b];
      }
      // measured (T = 64 vs 32 at config 2): the GEMM's time is additive in its store floor and its MMA
      // work -- operand loads and epilogue stores share the L2 -- so the constant store term does not
      // change the argmin and only the two variable terms are compared
      const double t_dense = head_cols * flops_per_col / rate;
      const double t = t_dense + tail_upd * t_atomic;
      if (best < 0 || t < best) { best = t; T = 1 << k; }
    }
    if (force_T >= 1) T = force_T;
  }
  int64_t Dc = 0, n_tail_cols = 0, n_tail_ent = 0;
  unsigned long long tail_work = 0;
  for (int b = 0; b < HIST_BUCKETS; ++b) {
    if (b < HIST_BUCKETS - 1 && (1LL << b) <= T) {
      n_tail_cols += (int64_t)hc.hist_cols[b];
      n_tail_ent += (int64_t)hc.hist_entries[b];
      tail_work += hc.hist_work[b];
    } else {
      Dc += (int64_t)hc.hist_cols[b];
    }
  }
  hc.T = T;
  if (getenv("GRAKEL_B200_DEBUG")) {
    fprintf(stderr, "[gk_gram] flops_per_col %.3g store_s %.3g T %d Dc %lld tail_cols %lld tail_ent %lld\n", flops_per_col,
            store_seconds, T, (long long)Dc, (long long)n_tail_cols, (long long)n_tail_ent);
    for (int b = 0; b < HIST_BUCKETS; ++b)
      fprintf(stderr, "  bucket %2d: cols %llu work %llu entries %llu\n", b, hc.hist_cols[b], hc.hist_work[b], hc.hist_entries[b]);
  }
  GK_TRY(h->tail_desc.ensure((size_t)std::max<int64_t>(n_tail_cols, 1) * sizeof(int2)));
  GK_TRY(h->tail_cur.ensure((size_t)std::max<int64_t>(n_tail_cols, 1) * 4));
  unsigned* col_counters = reinterpret_cast<unsigned*>(cs);  // the histogram has been read: reuse its first words
  GK_CUDA(cudaMemsetAsync(col_counters, 0, 16, h->stream));
  col_classify<<<nbc, 256, 0, h->stream>>>(D, square ? 1 : 0, (int)n_fit, fb.colcnt, h->colmin.as<int>(),
                                           h->colmax.as<int>(), T, h->colslot.as<int>(), h->tail_desc.as<int2>(),
                                           h->tail_cur.as<unsigned>(), col_counters);
  LAUNCH_CHECK(h);
  if (path == 1 && Dc == 0) path = 3;
  h->Dc = Dc;
  h->Dc_pad = (Dc + bk - 1) / bk * bk;
  if (force_T < 0 && path == 1 && square) h->head_row_bytes = h->Dc_pad * elem_bytes;

  // ---- transport type.  Tensor-core results are integers < 2^24 (checked above), i.e. exact in fp32: a float64
  // HOST result is produced and moved as fp32 (half the HBM writes; a quarter of the PCIe bytes for the
  // symmetric case, whose upper triangle alone is copied) and widened -- and, if asked, normalised in fp64 --
  // by host threads while the next band is in flight (host_deliver.h).  GRAKEL_B200_WIDEN=0 restores the
  // plain fp64 D2H copy of a device-side fp64 result.
  const char* widen_env = getenv("GRAKEL_B200_WIDEN");
  const bool widen_on_host = q.K_out && !(flags & GK_OUT_DEVICE) && out_dtype == GK_F64 && path != 2 &&
                             !(widen_env && atoi(widen_env) == 0);
  const bool host_norm = widen_on_host && normalize;
  const int32_t dev_dtype = widen_on_host ? GK_F32 : out_dtype;
  const size_t dev_esz = dev_dtype == GK_F64 ? 8 : 4;

  // multi-GPU row tiling (GK_DIST, collective): SYRK tiles shared between the ranks, mirrored halves stored into the
  // owner's row block over NVLink.  Needs the tensor path and fp32 device output; otherwise every rank computes its
  // row block with full tiles (the decision depends on replicated data only, so all ranks take the same branch).
  Comm* comm = reinterpret_cast<Comm*>(h->comm);
  const bool dist_req = (flags & (GK_DIST | GK_DIST_GATHER)) != 0;
  // GRAKEL_B200_DIST_SHARE=0: no tile sharing -- every rank computes its row block with full tiles (twice the SYRK
  // flops, no peer stores, no barriers): the round-1 scheme, kept for A/B measurements
  const char* e_share = getenv("GRAKEL_B200_DIST_SHARE");
  const bool dist = dist_req && path == 1 && dev_dtype == GK_F32 && !normalize && !(e_share && atoi(e_share) == 0);
  const bool gather = dist && (flags & GK_DIST_GATHER);
  const long long dist_per = dist_req ? dist_rows_per_rank(N, comm->nranks) : 0;


  // ---- output buffer
  void* d_out = nullptr;
  if (flags & GK_OUT_DEVICE) {
    d_out = q.K_out;
  } else {
    // library-owned K: rows padded to a multiple of 8 elements so that every row is 32-byte aligned
    // (TMA / 256-bit stores in the GEMM epilogue for any n_fit, e.g. 14 142 graphs on 2 GPUs)
    h->K_ld = (k_cols + 7) / 8 * 8;
    if (dist_req) {
      // the same request on every rank: a block of dist_per rows (all comm->nranks of them for the gathered result)
      const size_t blk = (size_t)dist_per * h->K_ld * dev_esz;
      GK_TRY(comm_share_K(h, (flags & GK_DIST_GATHER) ? blk * comm->nranks : blk));
      d_out = (flags & GK_DIST_GATHER) ? (void*)(h->K.as<char>() + (size_t)comm->rank * blk) : h->K.p;
    } else {
      GK_TRY(h->K.ensure((size_t)std::max<int64_t>(k_rows, 1) * h->K_ld * dev_esz));
      d_out = h->K.p;
    }
    h->K_rows = k_rows; h->K_cols = k_cols; h->K_dtype = dev_dtype;
  }
  const long long d_ld = (flags & GK_OUT_DEVICE) ? q.ld : h->K_ld;

  // panel-row ranges: A rows index K rows, B rows index K columns
  const int a0 = q.a0, a1 = q.a1;
  const int b0 = 0, b1 = (int)n_fit;
  const bool full_square = q.full_square;
  const bool mirror = (full_square && !(flags & GK_FULL_TILES)) || dist;
  const bool has_tail = path != 2 && n_tail_cols > 0;
  const bool norm_in_epilogue = normalize && !has_tail && !host_norm;

  GramParams p;
  memset(&p, 0, sizeof(p));
  p.a_row_end = a1; p.b_row_end = b1;
  p.c_row0 = a0; p.c_col0 = b0;
  p.out = d_out; p.ld = d_ld;
  p.mirror = mirror ? 1 : 0;
  p.fix_diag = square ? 1 : 0;
  p.nan_to_num = (flags & GK_NAN_TO_NUM) ? 1 : 0;
  p.vec_ok = (((uintptr_t)d_out) % 32 == 0 && (d_ld * (long long)dev_esz) % 32 == 0) ? 1 : 0;
  p.diag = h->diag_f64.as<double>();
  if (dist) {
    const size_t blk = (size_t)dist_per * d_ld * 4;
    for (int r = 0; r < comm->nranks; ++r)
      p.peer[r] = (flags & GK_DIST_GATHER) ? (void*)((char*)comm->peer_base[r] + (size_t)r * blk) : comm->peer_base[r];
    p.n_peers = comm->nranks;
    p.peer_rows = (int)dist_per;
  }
  if (dist) GK_TRY(comm_barrier(h));  // nobody still reads the block a peer is about to overwrite

  GK_CUDA(cudaEventRecord(h->tev[5], h->stream));
  int64_t n_tiles = 0;
  if (k_rows > 0) {
    // (always at least a stub: gk_wl_gram's asynchronous pass sizes its tail by the capacity left here)
    GK_TRY(h->tail_ent.ensure((size_t)std::max<int64_t>(has_tail ? n_tail_ent : 0, 64) * sizeof(int2)));
    if (path == 1 || path == 3) {
      const size_t panel_bytes = (size_t)N * std::max<int64_t>(h->Dc_pad, bk) * elem_bytes;
      GK_TRY(h->panel.ensure(panel_bytes));
      if (Dc) GK_CUDA(cudaMemsetAsync(h->panel.p, 0, panel_bytes, h->stream));
      if (Dc || has_tail) {
        if (elem_bytes == 1)
          feat_scatter<<<cdiv((long long)fb.cap, 256), 256, 0, h->stream>>>(
              fb.cap, fb.keys, fb.cnt, h->colslot.as<int>(), d_row_map,
              h->panel.as<uint8_t>(), h->Dc_pad, h->tail_cur.as<unsigned>(), h->tail_desc.as<int2>(),
              h->tail_ent.as<int2>());
        else
          feat_scatter<<<cdiv((long long)fb.cap, 256), 256, 0, h->stream>>>(
              fb.cap, fb.keys, fb.cnt, h->colslot.as<int>(), d_row_map,
              h->panel.as<__nv_bfloat16>(), h->Dc_pad, h->tail_cur.as<unsigned>(), h->tail_desc.as<int2>(),
              h->tail_ent.as<int2>());
        LAUNCH_CHECK(h);
      }
    }
    if (path == 1) {
      // cluster-pair kernel (gram_tc2.cuh: 256 x 256 tiles, the B tile multicast into both CTAs) for fp32
      // un-normalised output through TMA stores.  GRAKEL_B200_CTA2=0 selects the one-CTA kernel.
      const char* e_cta2 = getenv("GRAKEL_B200_CTA2");
      const bool cta2 = !(e_cta2 && atoi(e_cta2) == 0) && dev_dtype == GK_F32 && !norm_in_epilogue &&
                        ((uintptr_t)d_out) % 16 == 0 && (d_ld * 4) % 16 == 0 && !getenv("GRAKEL_B200_NO_TMA_STORE");
      if (dist && !cta2) return fail(GK_ERR_UNSUPPORTED, "gk_gram: GK_DIST needs the CTA-pair kernel (GRAKEL_B200_CTA2=0 is set?)");
      // the tile list depends on the shape of the request only: built and uploaded when that changes
      const long long tkey[8] = {dist ? 1 : 0, dist ? (long long)N : a0, dist ? comm->nranks : a1, dist ? comm->rank : b0, b1,
                                 mirror ? 1 : 0, cta2 ? BM2 : BM, 0};
      if (memcmp(tkey, h->tiles_key, sizeof(tkey)) != 0 || !h->tiles.p) {
        std::vector<int2> tiles;
        if (dist) dist_tiles(N, comm->nranks, comm->rank, tiles);
        else build_tiles(tiles, a0, a1, b0, b1, mirror, cta2 ? BM2 : BM);
        GK_TRY(h->h_tiles.ensure(tiles.size() * sizeof(int2) + 16));
        memcpy(h->h_tiles.p, tiles.data(), tiles.size() * sizeof(int2));
        GK_TRY(h->tiles.ensure(tiles.size() * sizeof(int2) + 16));
        GK_CUDA(cudaMemcpyAsync(h->tiles.p, h->h_tiles.p, tiles.size() * sizeof(int2), cudaMemcpyHostToDevice, h->stream));
        memcpy(h->tiles_key, tkey, sizeof(tkey));
        h->tiles_n = (long long)tiles.size();
      }
      n_tiles = h->tiles_n;
      CUtensorMap tmA, tmB, tmC;
      PeerMaps peer_maps;
      memset(&peer_maps, 0, sizeof(peer_maps));
      GK_TRY(make_panel_map(&tmA, h->panel.p, h->Dc_pad, N, BM, elem_bytes));
      GK_TRY(make_panel_map(&tmB, h->panel.p, h->Dc_pad, N, BN, elem_bytes));
      memset(&tmC, 0, sizeof(tmC));
      p.tma_store = 0;
      if (dev_dtype == GK_F32 && !norm_in_epilogue && ((uintptr_t)d_out) % 16 == 0 && (d_ld * 4) % 16 == 0 &&
          !getenv("GRAKEL_B200_NO_TMA_STORE")) {
        GK_TRY(make_out_map(&tmC, d_out, k_cols, k_rows, d_ld));
        p.tma_store = 1;
        if (p.mirror && !dist) {  // full square: the mirrored half goes through the same tensor map
          const char* e = getenv("GRAKEL_B200_MIRROR_TMA");
          if (!e || atoi(e) != 0) p.mirror = 2;
        }
        if (dist) {  // mirrored blocks as bulk TMA stores into the owners' row blocks (else 32 row stores of 128 B per block)
          const char* e = getenv("GRAKEL_B200_DIST_TMA");
          if (e && atoi(e) != 0) {
            for (int r = 0; r < comm->nranks; ++r) {
              const long long r_rows = std::min<long long>(N, (long long)(r + 1) * dist_per) - std::min<long long>(N, (long long)r * dist_per);
              if (r_rows > 0) GK_TRY(make_out_map(&peer_maps.m[r], p.peer[r], k_cols, r_rows, d_ld));
            }
            p.mirror = 2;
          }
        }
      }
      p.tiles = h->tiles.as<int2>();
      p.n_tiles = (int)n_tiles;
      p.num_k_blocks = (int)(h->Dc_pad / bk);
      const int grid = cta2 ? 2 * (int)std::min<int64_t>(n_tiles, h->sm_count / 2) : (int)std::min<int64_t>(n_tiles, h->sm_count);
      const bool prof = !cta2 && getenv("GRAKEL_B200_PROF") != nullptr;
      if (prof) {
        GK_TRY(h->K_stage.ensure((size_t)grid * 64));
        GK_CUDA(cudaMemsetAsync(h->K_stage.p, 0, (size_t)grid * 64, h->stream));
        p.prof = h->K_stage.as<long long>();
      }
      GK_CUDA(cudaEventRecord(h->tev[6], h->stream));
      if (n_tiles == 0) { /* a trailing rank without rows */ }
      else if (cta2 && elem_bytes == 1) gram_tc2_kernel<2><<<grid, GEMM_THREADS, GEMM2_SMEM, h->stream>>>(tmA, tmC, p, peer_maps);
      else if (cta2) gram_tc2_kernel<0><<<grid, GEMM_THREADS, GEMM2_SMEM, h->stream>>>(tmA, tmC, p, peer_maps);
      else if (dev_dtype == GK_F64) { if (norm_in_epilogue) launch_tc<double, true>(h, tmA, tmB, tmC, p, grid, elem_bytes); else launch_tc<double, false>(h, tmA, tmB, tmC, p, grid, elem_bytes); }
      else { if (norm_in_epilogue) launch_tc<float, true>(h, tmA, tmB, tmC, p, grid, elem_bytes); else launch_tc<float, false>(h, tmA, tmB, tmC, p, grid, elem_bytes); }
      LAUNCH_CHECK(h);
      if (prof) {
        std::vector<long long> pr((size_t)grid * 8);
        GK_CUDA(cudaMemcpyAsync(pr.data(), h->K_stage.p, pr.size() * 8, cudaMemcpyDeviceToHost, h->stream));
        GK_CUDA(cudaStreamSynchronize(h->stream));
        double a[8] = {0};
        for (int b = 0; b < grid; ++b) for (int i = 0; i < 8; ++i) a[i] += (double)pr[(size_t)b * 8 + i] / grid;
        fprintf(stderr, "[gram_tc prof] tiles %lld kblocks %d grid %d | consumers: epilogue %.0f wait_full %.0f total %.0f | tma: wait_empty %.0f total %.0f (avg cycles per CTA)\n",
                (long long)n_tiles, p.num_k_blocks, grid, a[0], a[1], a[4], a[5], a[6]);
      }
    } else if (path == 2) {
      const size_t panel_bytes = (size_t)N * std::max<int64_t>(Dc, 1) * 4;
      GK_TRY(h->panel.ensure(panel_bytes));
      GK_CUDA(cudaMemsetAsync(h->panel.p, 0, panel_bytes, h->stream));
      feat_fill_panel_u32<<<cdiv((long long)fb.cap, 256), 256, 0, h->stream>>>(
          fb.cap, fb.keys, fb.cnt, h->colslot.as<int>(), d_row_map,
          h->panel.as<unsigned>(), std::max<int64_t>(Dc, 1));
      LAUNCH_CHECK(h);
      GK_CUDA(cudaEventRecord(h->tev[6], h->stream));
      if (dev_dtype == GK_F64) { if (normalize) launch_simt<double, true>(h, h->panel.as<unsigned>(), std::max<int64_t>(Dc, 1), (int)Dc, a0, a1, b0, b1, p); else launch_simt<double, false>(h, h->panel.as<unsigned>(), std::max<int64_t>(Dc, 1), (int)Dc, a0, a1, b0, b1, p); }
      else { if (normalize) launch_simt<float, true>(h, h->panel.as<unsigned>(), std::max<int64_t>(Dc, 1), (int)Dc, a0, a1, b0, b1, p); else launch_simt<float, false>(h, h->panel.as<unsigned>(), std::max<int64_t>(Dc, 1), (int)Dc, a0, a1, b0, b1, p); }
      LAUNCH_CHECK(h);
    } else {
      GK_CUDA(cudaEventRecord(h->tev[6], h->stream));
      if (dev_dtype == GK_F64) { if (norm_in_epilogue) launch_empty<double, true>(h, a0, a1, b0, b1, p); else launch_empty<double, false>(h, a0, a1, b0, b1, p); }
      else { if (norm_in_epilogue) launch_empty<float, true>(h, a0, a1, b0, b1, p); else launch_empty<float, false>(h, a0, a1, b0, b1, p); }
      LAUNCH_CHECK(h);
    }
    GK_CUDA(cudaEventRecord(h->tev[7], h->stream));
    if (dist) GK_TRY(comm_barrier(h));  // the peers' mirrored stores into this block precede the tail's atomics
    if (has_tail) {
      const int grid = cdiv(n_tail_cols * 32, 256);
      if (dev_dtype == GK_F64)
        tail_pairs<double><<<grid, 256, 0, h->stream>>>(n_tail_cols, h->tail_desc.as<int2>(), h->tail_ent.as<int2>(),
                                                        (int)n_fit, square ? 1 : 0, (int)row_begin, (int)row_end,
                                                        (double*)d_out, d_ld);
      else
        tail_pairs<float><<<grid, 256, 0, h->stream>>>(n_tail_cols, h->tail_desc.as<int2>(), h->tail_ent.as<int2>(),
                                                       (int)n_fit, square ? 1 : 0, (int)row_begin, (int)row_end,
                                                       (float*)d_out, d_ld);
      LAUNCH_CHECK(h);
      if (normalize && !host_norm) {
        const double* drow = h->diag_f64.as<double>() + a0;
        const double* dcol = h->diag_f64.as<double>() + b0;
        if (dev_dtype == GK_F64)
          normalize_rows<double><<<h->sm_count * 8, 256, 0, h->stream>>>(k_rows, k_cols, (double*)d_out, d_ld, drow, dcol, p.nan_to_num);
        else
          normalize_rows<float><<<h->sm_count * 8, 256, 0, h->stream>>>(k_rows, k_cols, (float*)d_out, d_ld, drow, dcol, p.nan_to_num);
        LAUNCH_CHECK(h);
      }
    }
  } else {
    GK_CUDA(cudaEventRecord(h->tev[6], h->stream));
    GK_CUDA(cudaEventRecord(h->tev[7], h->stream));
    if (dist) GK_TRY(comm_barrier(h));
  }
  if (dist_req && (flags & GK_DIST_GATHER)) {
    // BASELINE config 4: every rank ends up with the full matrix -- one in-place all-gather of the finished row
    // blocks (NCCL over NVLink / NVSwitch); the library-owned result is reached through gk_result_device / gk_fetch
    NcclApi* api = nccl_api();
    const size_t cnt = (size_t)dist_per * d_ld;
    GK_CUDA(cudaEventRecord(h->ev[12], h->stream));
    GK_NCCL(api, api->AllGather(d_out, h->K.p, cnt, dev_dtype == GK_F64 ? ncclFloat64 : ncclFloat32, comm->comm, h->stream));
    h->K_rows = N;
  }
  GK_CUDA(cudaEventRecord(h->ev[13], h->stream));
  const int64_t launches_gram = h->launches - launches0;

  // ---- results to the host
  GK_CUDA(cudaEventRecord(h->ev[14], h->stream));
  if (q.K_out && !(flags & GK_OUT_DEVICE) && k_rows > 0) {
    if (widen_on_host) {
      const float* d_k = reinterpret_cast<const float*>(d_out);
      double* dst = reinterpret_cast<double*>(q.K_out);
      DeviceCopier cp{h};
      if (host_norm) {
        GK_TRY(h->h_diag.ensure((size_t)N * 8));
        GK_CUDA(cudaMemcpyAsync(h->h_diag.p, h->diag_f64.p, (size_t)N * 8, cudaMemcpyDeviceToHost, h->stream));
        GK_CUDA(cudaStreamSynchronize(h->stream));
        GK_TRY(deliver_rows(cp, d_k, d_ld, k_rows, k_cols, dst, q.ld, h->h_diag.as<double>() + a0, h->h_diag.as<double>() + b0,
                            p.nan_to_num));
      } else if (full_square && !getenv("GRAKEL_B200_NO_TRI")) {
        GK_TRY(deliver_square(h, d_k, d_ld, k_rows, dst, q.ld, max_diag));
      } else {
        GK_TRY(deliver_rows(cp, d_k, d_ld, k_rows, k_cols, dst, q.ld, nullptr, nullptr, 0));
      }
    } else {
      GK_CUDA(cudaMemcpy2DAsync(q.K_out, (size_t)q.ld * esz, d_out, (size_t)d_ld * esz, (size_t)k_cols * esz,
                                (size_t)k_rows, cudaMemcpyDeviceToHost, h->stream));
    }
  }
  if (q.xdiag) GK_CUDA(cudaMemcpyAsync(q.xdiag, h->diag_f64.p, n_fit * 8, cudaMemcpyDeviceToHost, h->stream));
  if (q.ydiag && !square)
    GK_CUDA(cudaMemcpyAsync(q.ydiag, h->diag_f64.as<double>() + n_fit, (N - n_fit) * 8, cudaMemcpyDeviceToHost, h->stream));
  GK_CUDA(cudaEventRecord(h->ev[15], h->stream));
  GK_CUDA(cudaStreamSynchronize(h->stream));
  if (stats) {
    stats->n_graphs = N; stats->n_vertices = h->V; stats->n_edges = h->E;
    stats->n_entries = n_entries;
    stats->n_dense_columns = Dc;
    stats->n_tail_columns = n_tail_cols;
    stats->tail_updates = (int64_t)tail_work;
    stats->threshold = hc.T;
    stats->max_count = max_count;
    stats->max_diag = max_diag;
    stats->gram_path = path;
    stats->gemm_elem_bytes = path == 1 && k_rows > 0 ? elem_bytes : 0;
    stats->gemm_tiles = n_tiles;
    stats->gemm_launches = launches_gram;
    stats->ms_panel = ev_ms(h->tev[4], h->tev[6]);
    stats->ms_gemm = ev_ms(h->tev[6], h->tev[7]);
    stats->ms_tail = ev_ms(h->tev[7], h->ev[13]);
    stats->ms_d2h = ev_ms(h->ev[14], h->ev[15]);
    stats->ms_total = ev_ms(h->tev[4], h->ev[15]);
  }
  return GK_OK;
}

// ---------------------------------------------------------------------------
// NeighborhoodSubgraphPairwiseDistance (nspd.cuh).  Level l = delta * (r + 1) + rho has its (graph, column) -> count
// table at nspd_blk + nspd_off[l]: keys [cap] u64 | counts [cap] u32 | graphs per column [M + 1] u32 | self
// similarities [N] u64 | largest count, entries (u32 x 2).
struct NspdLevel {
  unsigned long long* keys;
  unsigned* cnt;
  unsigned* colcnt;
  unsigned long long* diag;
  unsigned* part;
};

static size_t nspd_level_bytes(long long cap, long long M, long long N) {
  const size_t b = (size_t)cap * 12 + ((size_t)(M + 1) * 4 + 7) / 8 * 8 + (size_t)std::max<long long>(N, 1) * 8 + 8;
  return (b + 255) / 256 * 256;
}

static NspdLevel nspd_level(gk_handle* h, int l) {
  char* b = h->nspd_blk.as<char>() + h->nspd_off[l];
  const long long cap = h->nspd_cap[l], M = h->nspd_M[l];
  NspdLevel L;
  L.keys = reinterpret_cast<unsigned long long*>(b);
  L.cnt = reinterpret_cast<unsigned*>(b + cap * 8);
  L.colcnt = reinterpret_cast<unsigned*>(b + cap * 12);
  L.diag = reinterpret_cast<unsigned long long*>(b + cap * 12 + ((M + 1) * 4 + 7) / 8 * 8);
  L.part = reinterpret_cast<unsigned*>(L.diag + std::max<long long>(h->N, 1));
  return L;
}

// Host tables of gk_nspd_features, packed one after another (8-byte aligned) into nspd_aux.
struct NspdAux {
  std::vector<char> host;
  size_t add(const void* p, size_t bytes) {
    const size_t at = (host.size() + 7) / 8 * 8;
    host.resize(at + bytes);
    if (bytes) memcpy(host.data() + at, p, bytes);
    return at;
  }
};

static int nspd_build_params(gk_handle* h, const int64_t* sym_hash, const int32_t* edge_label, const int32_t* tok_rank,
                             int64_t n_labels, const int64_t* rank_off, const uint8_t* rank_bytes, const int32_t* rank_cp,
                             int32_t n_ranks, const int64_t* el_off, const uint8_t* el_bytes, const int32_t* el_cp,
                             int32_t n_elabels, NspdParams* p, std::vector<long long>* lvl_off_h) {
  const int64_t N = h->N, V = h->V, E = h->E;
  const std::vector<int>& gp = h->graph_ptr_host;
  lvl_off_h->assign(N + 1, 0);
  for (int64_t g = 0; g < N; ++g) {
    const long long n = gp[g + 1] - gp[g];
    (*lvl_off_h)[g + 1] = (*lvl_off_h)[g] + n * n;
  }
  NspdAux a;
  const size_t o_sym = a.add(sym_hash, (size_t)V * 8);
  const size_t o_el = a.add(edge_label, (size_t)E * 4);
  const size_t o_tok = a.add(tok_rank, (size_t)(h->nspd_d + 1) * n_labels * 4);
  const size_t o_roff = a.add(rank_off, (size_t)(n_ranks + 1) * 8);
  const size_t o_rb = a.add(rank_bytes, (size_t)rank_off[n_ranks]);
  const size_t o_rcp = a.add(rank_cp, (size_t)n_ranks * 4);
  const size_t o_eoff = a.add(el_off, (size_t)(n_elabels + 1) * 8);
  const size_t o_eb = a.add(el_bytes, (size_t)el_off[n_elabels]);
  const size_t o_ecp = a.add(el_cp, (size_t)n_elabels * 4);
  const size_t o_loff = a.add(lvl_off_h->data(), (size_t)(N + 1) * 8);
  std::vector<unsigned char> loop(std::max<int64_t>(V, 1), 0);
  {
    std::vector<int> rp(V + 1), ci(std::max<int64_t>(E, 1));
    GK_CUDA(cudaMemcpy(rp.data(), h->row_ptr.p, (V + 1) * 4, cudaMemcpyDeviceToHost));
    if (E) GK_CUDA(cudaMemcpy(ci.data(), h->col_idx.p, E * 4, cudaMemcpyDeviceToHost));
    for (int64_t v = 0; v < V; ++v)
      for (int k = rp[v]; k < rp[v + 1]; ++k)
        if (ci[k] == v) loop[v] = 1;
  }
  const size_t o_loop = a.add(loop.data(), (size_t)V);
  GK_TRY(h->nspd_aux.ensure(a.host.size() + 8));
  GK_CUDA(cudaMemcpy(h->nspd_aux.p, a.host.data(), a.host.size(), cudaMemcpyHostToDevice));
  char* d = h->nspd_aux.as<char>();
  memset(p, 0, sizeof(*p));
  p->N = (int)N; p->r = h->nspd_r; p->d = h->nspd_d; p->n_labels = (int)n_labels;
  p->graph_ptr = h->graph_ptr.as<int>(); p->row_ptr = h->row_ptr.as<int>(); p->col_idx = h->col_idx.as<int>();
  p->labels = h->labels0.as<int>();
  p->edge_label = reinterpret_cast<const int*>(d + o_el);
  p->sym_hash = reinterpret_cast<const long long*>(d + o_sym);
  p->lvl_off = reinterpret_cast<const long long*>(d + o_loff);
  p->tok_rank = reinterpret_cast<const int*>(d + o_tok);
  p->rank_off = reinterpret_cast<const long long*>(d + o_roff);
  p->rank_bytes = reinterpret_cast<const unsigned char*>(d + o_rb);
  p->rank_cp = reinterpret_cast<const int*>(d + o_rcp);
  p->el_off = reinterpret_cast<const long long*>(d + o_eoff);
  p->el_bytes = reinterpret_cast<const unsigned char*>(d + o_eb);
  p->el_cp = reinterpret_cast<const int*>(d + o_ecp);
  p->selfloop = reinterpret_cast<const unsigned char*>(d + o_loop);
  return GK_OK;
}

extern "C" {

int gk_nspd_features(gk_handle* h, int32_t r, int32_t d, const int64_t* sym_hash, const int32_t* edge_label,
                     const int32_t* tok_rank, int64_t n_labels, const int64_t* rank_off, const uint8_t* rank_bytes,
                     const int32_t* rank_cp, int32_t n_ranks, const int64_t* el_off, const uint8_t* el_bytes,
                     const int32_t* el_cp, int32_t n_elabels, uint64_t* delta_mask, int32_t flags, gk_stats* stats) {
  GK_TRY(need_packed(h, "gk_nspd_features"));
  if (!h->has_labels) return fail(GK_ERR_ARG, "gk_nspd_features: vertex labels are required");
  if (r < 0 || d < 0) return fail(GK_ERR_ARG, "gk_nspd_features: r and d must be >= 0");
  if ((int64_t)(r + 1) * (d + 1) > MAX_LEVELS)
    return fail(GK_ERR_UNSUPPORTED, "gk_nspd_features: (r + 1)(d + 1) levels exceed 64");
  if (flags != 0) return fail(GK_ERR_ARG, "gk_nspd_features: no flags are defined");
  if (!sym_hash || (!edge_label && h->E) || !tok_rank || !rank_off || !rank_cp || !el_off || (!el_cp && n_elabels))
    return fail(GK_ERR_ARG, "gk_nspd_features: null table");
  if (n_labels < h->n_labels0) return fail(GK_ERR_ARG, "gk_nspd_features: a token is needed for every label id");
  const int64_t N = h->N, V = h->V, E = h->E;
  const int64_t launches0 = h->launches;
  features_begin(h);
  const std::vector<int>& gp = h->graph_ptr_host;
  long long max_n = 1, max_e = 1;
  for (int64_t g = 0; g < N; ++g) {
    max_n = std::max<long long>(max_n, gp[g + 1] - gp[g]);
    max_e = std::max<long long>(max_e, h->graph_eptr_host[g + 1] - h->graph_eptr_host[g]);
  }
  // refused before any table is sized: the level matrices alone take 5 n^2 bytes per graph
  const long long ball = r > 0 ? max_n + 1 : 1;
  if (ball * ball >= (1LL << 32))  // label offsets are u32
    return fail(GK_ERR_UNSUPPORTED, "gk_nspd_features: r > 0 with a graph of 65535 or more vertices");
  h->nspd_r = r; h->nspd_d = d;
  GK_TRY(init_scalars(h, 0));
  GK_CUDA(cudaEventRecord(h->tev[2], h->stream));
  NspdParams p;
  std::vector<long long> loff;
  GK_TRY(nspd_build_params(h, sym_hash, edge_label, tok_rank, n_labels, rank_off, rank_bytes, rank_cp, n_ranks, el_off,
                           el_bytes, el_cp, n_elabels, &p, &loff));
  const long long P = loff[N];
  // ---- BFS levels
  GK_TRY(h->nspd_lvl.ensure((size_t)std::max<long long>(P, 1)));
  GK_TRY(h->nspd_q.ensure((size_t)std::max<long long>(P, 1) * 4));
  p.lvl = h->nspd_lvl.as<unsigned char>();
  const int max_level = r > 0 ? std::max(r, d) : 0;
  nspd_bfs<<<cdiv(V, 128), 128, 0, h->stream>>>((int)V, (int)N, p.graph_ptr, p.row_ptr, p.col_idx, p.lvl_off, max_level,
                                                h->nspd_lvl.as<unsigned char>(), h->nspd_q.as<int>());
  LAUNCH_CHECK(h);
  // ---- hashes: one slot per vertex, fewer under the workspace budget (GRAKEL_B200_NSPD_WS_BUDGET=<bytes>)
  GK_TRY(h->nspd_H.ensure((size_t)(r + 1) * std::max<int64_t>(V, 1) * 4));
  p.H = h->nspd_H.as<unsigned>();
  p.set_cap = (long long)nspd_set_cap(max_e);
  p.max_e = max_e;
  p.max_n = max_n;
  p.ball = ball;
  p.slot_words = nspd_slot_words(p.set_cap, max_e, max_n, p.ball);
  size_t budget = (size_t)4 << 30;
  if (const char* e = getenv("GRAKEL_B200_NSPD_WS_BUDGET")) budget = std::max<size_t>(1, strtoull(e, nullptr, 10));
  const long long slots = std::max<long long>(1, std::min<long long>(V, (long long)(budget / ((size_t)p.slot_words * 4))));
  p.n_slots = (int)slots;
  GK_TRY(h->nspd_ws.ensure((size_t)slots * p.slot_words * 4));
  p.ws = h->nspd_ws.as<unsigned>();
  nspd_hash<<<cdiv(slots, 64), 64, 0, h->stream>>>(p, (int)V);
  LAUNCH_CHECK(h);
  GK_CUDA(cudaEventRecord(h->tev[6], h->stream));
  // ---- pairs of every distance: count, then fill
  const int D1 = d + 1;
  GK_TRY(h->nspd_keys.ensure((size_t)(3 * D1 + N) * 8 + 64));
  unsigned long long* cnt = h->nspd_keys.as<unsigned long long>();
  unsigned long long* cursor = cnt + D1;
  unsigned long long* base = cursor + D1;
  unsigned long long* mask = base + D1;
  GK_CUDA(cudaMemsetAsync(cnt, 0, (size_t)(3 * D1 + N) * 8, h->stream));
  const int pgrid = (int)std::min<int64_t>(N, (int64_t)h->sm_count * 16);
  nspd_pairs<<<pgrid, 256, 0, h->stream>>>((int)N, r, d, p.graph_ptr, p.lvl_off, p.lvl, p.selfloop, 0, cnt, cursor, base,
                                           nullptr, nullptr, mask);
  LAUNCH_CHECK(h);
  std::vector<unsigned long long> hc(D1 + N);
  GK_CUDA(cudaMemcpyAsync(hc.data(), cnt, D1 * 8, cudaMemcpyDeviceToHost, h->stream));
  GK_CUDA(cudaMemcpyAsync(hc.data() + D1, mask, N * 8, cudaMemcpyDeviceToHost, h->stream));
  GK_CUDA(cudaStreamSynchronize(h->stream));
  std::vector<unsigned long long> hb(D1, 0);
  unsigned long long tot = 0, Mmax = 1;
  for (int t = 0; t < D1; ++t) { hb[t] = tot; tot += hc[t]; Mmax = std::max(Mmax, hc[t]); }
  if (tot >= (1ULL << 31)) return fail(GK_ERR_UNSUPPORTED, "gk_nspd_features: 2^31 or more vertex pairs");
  h->nspd_mask.assign(hc.begin() + D1, hc.end());
  if (delta_mask) memcpy(delta_mask, h->nspd_mask.data(), N * 8);
  GK_TRY(h->nspd_pairs.ensure((size_t)std::max<unsigned long long>(tot, 1) * 8));
  unsigned* A = h->nspd_pairs.as<unsigned>();
  unsigned* Bv = A + std::max<unsigned long long>(tot, 1);
  GK_CUDA(cudaMemcpyAsync(base, hb.data(), D1 * 8, cudaMemcpyHostToDevice, h->stream));
  nspd_pairs<<<pgrid, 256, 0, h->stream>>>((int)N, r, d, p.graph_ptr, p.lvl_off, p.lvl, p.selfloop, 1, cnt, cursor, base,
                                           A, Bv, mask);
  LAUNCH_CHECK(h);
  // ---- per-level tables (delta-major), numbered with the NeighborhoodHash column passes
  const int n_lev = D1 * (r + 1);
  h->nspd_off.assign(n_lev, 0); h->nspd_cap.assign(n_lev, 0); h->nspd_M.assign(n_lev, 0); h->nspd_cols.assign(n_lev, 0);
  size_t blk = 0;
  for (int l = 0; l < n_lev; ++l) {
    const long long M = (long long)hc[l / (r + 1)];
    h->nspd_M[l] = M;
    h->nspd_cap[l] = (long long)std::max<size_t>(next_pow2((size_t)std::max<long long>(M, 1) * 2), 1024);
    h->nspd_off[l] = (long long)blk;
    blk += nspd_level_bytes(h->nspd_cap[l], M, N);
  }
  GK_TRY(h->nspd_blk.ensure(blk));
  const size_t tcap = std::max<size_t>(next_pow2((size_t)Mmax * 2), 1024);
  GK_TRY(h->nspd_tab.ensure(tcap * 8 + (size_t)Mmax * 4));
  int* tab = h->nspd_tab.as<int>();
  int* colid = tab + tcap;
  int* slot_of = colid + tcap;
  GK_TRY(h->nspd_C.ensure((size_t)Mmax * 13 + (size_t)n_lev * 8 + 64));  // keys | entry graphs | valid | columns
  unsigned long long* keys = h->nspd_C.as<unsigned long long>();
  int* egraph = reinterpret_cast<int*>(keys + Mmax);
  unsigned char* valid = reinterpret_cast<unsigned char*>(egraph + Mmax);
  unsigned long long* dims = reinterpret_cast<unsigned long long*>(h->nspd_C.as<char>() + ((size_t)Mmax * 13 + 7) / 8 * 8);
  GK_CUDA(cudaMemsetAsync(valid, 1, Mmax, h->stream));
  GK_CUDA(cudaMemsetAsync(dims, 0, (size_t)n_lev * 8, h->stream));
  GK_CUDA(cudaMemsetAsync(h->nspd_blk.p, 0, blk, h->stream));
  for (int l = 0; l < n_lev; ++l) {
    const int delta = l / (r + 1), rho = l % (r + 1);
    const long long M = h->nspd_M[l];
    const size_t cap = (size_t)h->nspd_cap[l];
    NspdLevel L = nspd_level(h, l);
    GK_CUDA(cudaMemsetAsync(L.keys, 0xFF, cap * 8, h->stream));
    if (!M) continue;
    nspd_keys<<<cdiv(M, 256), 256, 0, h->stream>>>(M, A + hb[delta], Bv + hb[delta], p.H + (size_t)rho * V,
                                                   h->vgraph.as<int>(), keys, egraph);
    LAUNCH_CHECK(h);
    GK_CUDA(cudaMemsetAsync(tab, 0xFF, tcap * 4, h->stream));
    nh_code_insert<<<cdiv(M, 256), 256, 0, h->stream>>>((int)M, keys, valid, tab, (unsigned)(tcap - 1), slot_of);
    LAUNCH_CHECK(h);
    nh_code_number<<<cdiv(M, 256), 256, 0, h->stream>>>((int)M, valid, tab, slot_of, colid, dims + l);
    LAUNCH_CHECK(h);
    nh_count<<<cdiv(M, 256), 256, 0, h->stream>>>((int)M, 1, valid, egraph, slot_of, colid, L.keys, L.cnt,
                                                  (unsigned)(cap - 1));
    LAUNCH_CHECK(h);
    nspd_level_stats<<<cdiv((long long)cap, 256), 256, 0, h->stream>>>(cap, L.keys, L.cnt, L.colcnt, L.diag, L.part);
    LAUNCH_CHECK(h);
  }
  GK_CUDA(cudaEventRecord(h->tev[3], h->stream));
  std::vector<unsigned long long> hd(n_lev);
  GK_CUDA(cudaMemcpyAsync(hd.data(), dims, n_lev * 8, cudaMemcpyDeviceToHost, h->stream));
  GK_CUDA(cudaStreamSynchronize(h->stream));
  int64_t n_cols = 0;
  for (int l = 0; l < n_lev; ++l) { h->nspd_cols[l] = (long long)hd[l]; n_cols += (int64_t)hd[l]; }
  h->n_columns = n_cols;
  features_publish(h, FK_NSPD);
  if (stats) {
    memset(stats, 0, sizeof(*stats));
    stats->n_graphs = N; stats->n_vertices = V; stats->n_edges = E;
    stats->n_levels = n_lev;
    for (int l = 0; l < n_lev; ++l) stats->level_dims[l] = h->nspd_cols[l];
    stats->n_columns = n_cols;
    stats->n_entries = (int64_t)tot;
    stats->kernel_launches = h->launches - launches0;
    stats->ms_features = ev_ms(h->tev[2], h->tev[3]);
    stats->ms_hash = ev_ms(h->tev[2], h->tev[6]);
    stats->ms_columns = ev_ms(h->tev[6], h->tev[3]);
  }
  return GK_OK;
}

int gk_nspd_hashes(gk_handle* h, int32_t radius, uint32_t* out) {
  if (!h || !out) return fail(GK_ERR_ARG, "gk_nspd_hashes: null argument");
  if (h->feature_kind != FK_NSPD || radius < 0 || radius > h->nspd_r)
    return fail(GK_ERR_STATE, "gk_nspd_hashes: no such radius (run gk_nspd_features first)");
  GK_CUDA(cudaSetDevice(h->dev));
  if (h->V) {
    GK_CUDA(cudaMemcpyAsync(out, h->nspd_H.as<unsigned>() + (size_t)radius * h->V, (size_t)h->V * 4,
                            cudaMemcpyDeviceToHost, h->stream));
    GK_CUDA(cudaStreamSynchronize(h->stream));
  }
  return GK_OK;
}

// CPython's set on n distinct pairs inserted in order (element hashes h0[k], h1[k]); order[] = iteration order.
int gk_selftest_nspd_set_order(int64_t n, const int64_t* h0, const int64_t* h1, int64_t* order) {
  if (n < 0 || (n && (!h0 || !h1 || !order))) return fail(GK_ERR_ARG, "gk_selftest_nspd_set_order: bad argument");
  const unsigned long long cap = nspd_set_cap(n);
  std::vector<unsigned> buf(2 * cap);
  NspdSet s;
  s.buf[0] = buf.data();
  s.buf[1] = buf.data() + cap;
  nspd_set_clear(s);
  auto hash_of = [&](unsigned id) { return nspd_tuple_hash(h0[id], h1[id]); };
  for (int64_t k = 0; k < n; ++k) nspd_set_add(s, (unsigned)k, hash_of((unsigned)k), hash_of);
  int64_t m = 0;
  for (unsigned long long k = 0; k <= s.mask; ++k)
    if (s.buf[s.cur][k] != NSPD_EMPTY) order[m++] = s.buf[s.cur][k];
  return m == n ? GK_OK : fail(GK_ERR_STATE, "gk_selftest_nspd_set_order: lost an item");
}

}  // extern "C"

// Gram of NeighborhoodSubgraphPairwiseDistance features (gram_path 12): per level, in the reference's order, the
// exact integer Gram of its count table as fp64 counts, folded into K at once (one count matrix live).  The levels
// are those the fitted graphs have (square case) or that both sides have (transform); GK_NORMALIZE divides by the
// number of fitted levels, or by sqrt(levels of Y x levels of X).  Rows go in chunks when one level's count matrix of
// the whole request would exceed 8 GiB (GRAKEL_B200_NSPD_C_BUDGET=<bytes> lowers it).
static int gram_nspd(gk_handle* h, const GramReq& q, gk_stats* stats) {
  const int64_t N = h->N, n_fit = q.n_fit, k_rows = q.k_rows, k_cols = q.k_cols;
  const bool square = q.square;
  const int r1 = h->nspd_r + 1;
  const int64_t launches0 = h->launches;
  auto maxd = [&](int64_t a, int64_t b) {
    int m = -1;
    for (int64_t g = a; g < b; ++g)
      if (h->nspd_mask[g]) m = std::max(m, 63 - __builtin_clzll(h->nspd_mask[g]));
    return m;
  };
  const int mx = maxd(0, n_fit), my = square ? mx : maxd(n_fit, N);
  const int m_use = std::min(mx, my);
  const long long nlx = (long long)r1 * (mx + 1), nly = (long long)r1 * (my + 1);
  F64Out out;
  GK_TRY(f64_target(h, q, &out));
  const int64_t ldc = (k_cols + 7) / 8 * 8;
  size_t c_budget = (size_t)8 << 30;
  if (const char* e = getenv("GRAKEL_B200_NSPD_C_BUDGET")) c_budget = std::max<size_t>(1, strtoull(e, nullptr, 10));
  const int64_t chunk = std::max<int64_t>(1, std::min<int64_t>(std::max<int64_t>(k_rows, 1), (int64_t)(c_budget / ((size_t)ldc * 8))));
  GK_TRY(h->nh_C.ensure((size_t)chunk * ldc * 8));
  double* C = h->nh_C.as<double>();
  const int32_t gflags = (q.flags & (GK_GRAM_SIMT | GK_DENSE_ALL)) | GK_FULL_TILES | GK_OUT_DEVICE;
  std::vector<float> ms_level(64, 0.f);
  float ms_fold = 0.f;
  int64_t max_T = 0, gram_launches = 0, elem_bytes = 0;
  for (int64_t cb = q.row_begin; cb < q.row_end; cb += chunk) {
    const int64_t ce = std::min<int64_t>(q.row_end, cb + chunk), rows = ce - cb;
    double* o = out.p + (size_t)(cb - q.row_begin) * out.ld;
    GK_CUDA(cudaMemset2DAsync(o, (size_t)out.ld * 8, 0, (size_t)k_cols * 8, (size_t)rows, h->stream));
    for (int delta = 0; delta <= m_use; ++delta)
      for (int rho = 0; rho < r1; ++rho) {
        const int l = delta * r1 + rho;
        NspdLevel L = nspd_level(h, l);
        IntBlock fb;
        fb.keys = L.keys; fb.cnt = L.cnt; fb.cap = (size_t)h->nspd_cap[l];
        fb.colcnt = L.colcnt; fb.col_cap = h->nspd_M[l] + 1; fb.n_columns = h->nspd_cols[l];
        fb.diag = L.diag; fb.part_max = L.part; fb.part_new = L.part + 1; fb.n_part = 1;
        fb.prologue_on_host = false;
        GramReq lq;
        GK_TRY(gram_request(h, FK_WL, n_fit, gflags, cb, ce, C, GK_F64, ldc, nullptr, nullptr, &lq));
        gk_stats st;
        memset(&st, 0, sizeof(st));
        GK_TRY(gram_int(h, lq, fb, &st));
        ms_level[l] += st.ms_total;
        max_T = std::max<int64_t>(max_T, st.threshold);
        gram_launches += st.gemm_launches;
        elem_bytes = std::max<int64_t>(elem_bytes, st.gemm_elem_bytes);
        if (rows > 0) {
          GK_CUDA(cudaEventRecord(h->tev[0], h->stream));
          nspd_fold<<<cdiv(rows * k_cols, 256), 256, 0, h->stream>>>((int)rows, (int)k_cols, C, ldc,
                                                                     (int)((square ? 0 : n_fit) + cb), L.diag,
                                                                     square ? 1 : 0, o, out.ld);
          LAUNCH_CHECK(h);
          GK_CUDA(cudaEventRecord(h->tev[1], h->stream));
          GK_CUDA(cudaEventSynchronize(h->tev[1]));
          ms_fold += ev_ms(h->tev[0], h->tev[1]);
        }
      }
    if ((q.flags & GK_NORMALIZE) && rows > 0) {
      const double div = square ? (double)nlx : sqrt((double)nly * (double)nlx);
      nspd_scale<<<cdiv(rows * k_cols, 256), 256, 0, h->stream>>>((int)rows, (int)k_cols, div, o, out.ld);
      LAUNCH_CHECK(h);
    }
  }
  GramReq kq = q;  // diagonal(): the number of levels of each side, written on the host
  kq.xdiag = kq.ydiag = nullptr;
  GK_TRY(f64_deliver(h, kq, out, false, h->ev[14], h->ev[15]));
  if (q.xdiag) for (int64_t i = 0; i < n_fit; ++i) q.xdiag[i] = (double)nlx;
  if (q.ydiag && !square) for (int64_t i = 0; i < N - n_fit; ++i) q.ydiag[i] = (double)nly;
  if (stats) {
    stats->n_graphs = N; stats->n_vertices = h->V; stats->n_edges = h->E;
    stats->n_levels = (int64_t)r1 * (m_use + 1);
    stats->gram_path = 12;
    stats->threshold = max_T;
    stats->gemm_launches = gram_launches + (h->launches - launches0);
    stats->gemm_elem_bytes = elem_bytes;
    float tot = ms_fold;
    for (int l = 0; l < 64; ++l) { stats->ms_level_gram[l] = ms_level[l]; tot += ms_level[l]; }
    stats->ms_gemm = tot - ms_fold;
    stats->ms_combine = ms_fold;
    stats->ms_d2h = ev_ms(h->ev[14], h->ev[15]);
    stats->ms_total = tot + stats->ms_d2h;
  }
  return GK_OK;
}

static int gram_odd(gk_handle* h, const GramReq& q, gk_stats* stats);
static int gram_ml(gk_handle* h, const GramReq& q, gk_stats* stats);
static int gram_svmt(gk_handle* h, const GramReq& q, gk_stats* stats);
static int gram_gs(gk_handle* h, const GramReq& q, gk_stats* stats);

// The route of the packed feature kind: gk_gram and gk_core_level_add.
static int gram_route(gk_handle* h, const GramReq& q, gk_stats* stats) {
  switch (h->feature_kind) {
    case FK_SPATTR: return gram_spattr(h, q, stats);
    case FK_GH: return h->gh_node_kernel == GK_GH_LINEAR ? gram_spattr(h, q, stats) : gram_gh_nodepair(h, q, stats);
    case FK_NH: return gram_nh(h, q, stats);
    case FK_PM: return gram_pm(h, q, stats);
    case FK_NSPD: return gram_nspd(h, q, stats);
    case FK_RW: return gram_rw(h, q, stats);
    case FK_SM: return gram_sm(h, q, stats);
    case FK_ODD: return gram_odd(h, q, stats);
    case FK_ML: return gram_ml(h, q, stats);
    case FK_SVMT: return gram_svmt(h, q, stats);
    case FK_GS: return gram_gs(h, q, stats);
    default: return gram_int(h, q, block_of(h), stats);
  }
}

// ---------------------------------------------------------------------------
// WL over NeighborhoodSubgraphPairwiseDistance.  Every WL level's K is itself a sum of cosine-normalised per-(radius,
// distance) Grams, so the WL levels cannot share one feature block: the host packs each level's labels and runs
// gk_nspd_features, gk_wl_level_sum folds that level's K (gram_nspd, un-normalised) and adds it into a running sum on
// the device, in level order, and gk_wl_level_sum_fetch normalises the sum and copies it out.
extern "C" {

int gk_wl_level_sum(gk_handle* h, int32_t level, int64_t n_fit, int64_t row_begin, int64_t row_end, gk_stats* stats) {
  if (!h) return fail(GK_ERR_ARG, "null handle");
  if (h->feature_kind != FK_NSPD)
    return fail(GK_ERR_STATE, "gk_wl_level_sum: run gk_nspd_features on the level's labels first");
  if (level < 0 || (level > 0 && (level != h->wl_sum_levels || h->core_sum)))
    return fail(GK_ERR_ARG, "gk_wl_level_sum: levels must be added in order, starting at 0");
  GramReq q;
  GK_TRY(gram_request(h, FK_NSPD, n_fit, 0, row_begin, row_end, nullptr, GK_F64, 0, nullptr, nullptr, &q));
  if (level > 0 && (q.k_rows != h->wl_sum_rows || q.k_cols != h->wl_sum_cols || q.square != h->wl_sum_square ||
                    q.row_begin != h->wl_sum_row0))
    return fail(GK_ERR_ARG, "gk_wl_level_sum: a level's K has another shape than the sum's");
  GK_CUDA(cudaSetDevice(h->dev));
  const size_t elems = (size_t)q.k_rows * q.k_cols;
  gk::DevBuf& dst = level == 0 ? h->wl_sum : h->wl_lvl;
  GK_TRY(dst.ensure(std::max<size_t>(elems, 1) * 8));
  q.flags |= GK_OUT_DEVICE; q.dev_out = true; q.K_out = dst.p; q.ld = q.k_cols;
  GK_TRY(gram_nspd(h, q, stats));
  if (level > 0 && elems) {
    add_f64<<<(int)std::min<size_t>((elems + 255) / 256, (size_t)h->sm_count * 16), 256, 0, h->stream>>>(
        (long long)elems, h->wl_lvl.as<double>(), h->wl_sum.as<double>());
    LAUNCH_CHECK(h);
  }
  h->wl_sum_rows = q.k_rows; h->wl_sum_cols = q.k_cols; h->wl_sum_row0 = q.row_begin; h->wl_sum_square = q.square;
  h->wl_sum_levels = level + 1;
  h->core_sum = false;
  GK_CUDA(cudaStreamSynchronize(h->stream));
  return GK_OK;
}

int gk_wl_level_sum_fetch(gk_handle* h, int32_t flags, const double* xdiag, const double* ydiag, double* K_out,
                          double* kdiag) {
  if (!h) return fail(GK_ERR_ARG, "null handle");
  if (h->wl_sum_levels <= 0 && !h->core_sum)
    return fail(GK_ERR_STATE, "gk_wl_level_sum_fetch: no level added (gk_wl_level_sum) and no gk_core_sum_begin");
  if (flags & ~(GK_NORMALIZE | GK_NAN_TO_NUM)) return fail(GK_ERR_ARG, "gk_wl_level_sum_fetch: unknown flags");
  GK_CUDA(cudaSetDevice(h->dev));
  const int64_t rows = h->wl_sum_rows, cols = h->wl_sum_cols;
  const bool full_square = h->wl_sum_square && h->wl_sum_row0 == 0 && rows == cols;
  double* K = h->wl_sum.as<double>();
  GK_TRY(h->diag_f64.ensure((size_t)(rows + cols + 1) * 8));
  double* dcol = h->diag_f64.as<double>();
  double* drow = dcol + cols;
  if (kdiag || ((flags & GK_NORMALIZE) && !xdiag)) {
    if (!full_square) return fail(GK_ERR_ARG, "gk_wl_level_sum_fetch: the diagonal of K needs the full square sum");
    if (cols) {
      diag_of_f64<<<cdiv(cols, 256), 256, 0, h->stream>>>(cols, K, cols, dcol);
      LAUNCH_CHECK(h);
    }
    if (kdiag) GK_CUDA(cudaMemcpyAsync(kdiag, dcol, (size_t)cols * 8, cudaMemcpyDeviceToHost, h->stream));
  }
  if ((flags & GK_NORMALIZE) && rows > 0) {
    const double* dr = dcol;
    if (xdiag) {  // the caller's self similarities: xdiag for the columns, ydiag (or xdiag's rows) for the rows
      GK_CUDA(cudaMemcpyAsync(dcol, xdiag, (size_t)cols * 8, cudaMemcpyHostToDevice, h->stream));
      if (h->wl_sum_square) {
        dr = dcol + h->wl_sum_row0;
      } else {
        if (!ydiag) return fail(GK_ERR_ARG, "gk_wl_level_sum_fetch: a transform needs ydiag to normalise");
        GK_CUDA(cudaMemcpyAsync(drow, ydiag + h->wl_sum_row0, (size_t)rows * 8, cudaMemcpyHostToDevice, h->stream));
        dr = drow;
      }
    } else {
      dr = dcol;
    }
    normalize_rows<double><<<h->sm_count * 8, 256, 0, h->stream>>>(rows, cols, K, cols, dr, dcol,
                                                                    (flags & GK_NAN_TO_NUM) ? 1 : 0);
    LAUNCH_CHECK(h);
  }
  if (K_out && rows > 0) GK_CUDA(cudaMemcpyAsync(K_out, K, (size_t)rows * cols * 8, cudaMemcpyDeviceToHost, h->stream));
  GK_CUDA(cudaStreamSynchronize(h->stream));
  return GK_OK;
}

}  // extern "C"

// ---------------------------------------------------------------------------
// CoreFramework over a base kernel whose core levels cannot share one feature block (NeighborhoodHash, OddSth,
// WeisfeilerLehmanOptimalAssignment, SubgraphMatching).  The reference fits one base kernel per core level and adds
// its K into the rows and columns of the graphs that have that level's subgraph, K[idx_j, idx] += K_i[j, :], from the
// largest core down (core_framework.py:177-223).  gk_core_sum_begin zeroes the sum (the wl_sum buffer of
// gk_wl_level_sum), gk_core_level_add computes one level's un-normalised K on the device (wl_lvl) and scatters it into
// the sum, and gk_wl_level_sum_fetch normalises and copies the sum out once.
extern "C" {

int gk_core_sum_begin(gk_handle* h, int64_t n_rows, int64_t n_cols, int32_t square) {
  if (!h) return fail(GK_ERR_ARG, "null handle");
  if (n_rows < 0 || n_cols <= 0 || n_rows > INT32_MAX || n_cols > INT32_MAX)
    return fail(GK_ERR_ARG, "gk_core_sum_begin: bad shape");
  if (square && n_rows != n_cols) return fail(GK_ERR_ARG, "gk_core_sum_begin: a square sum needs n_rows == n_cols");
  GK_CUDA(cudaSetDevice(h->dev));
  const size_t elems = (size_t)n_rows * (size_t)n_cols;
  GK_TRY(h->wl_sum.ensure(std::max<size_t>(elems, 1) * 8));
  if (elems) GK_CUDA(cudaMemsetAsync(h->wl_sum.p, 0, elems * 8, h->stream));
  h->wl_sum_rows = n_rows; h->wl_sum_cols = n_cols; h->wl_sum_row0 = 0; h->wl_sum_square = square != 0;
  h->wl_sum_levels = 0;
  h->core_sum = true;
  h->core_level = INT32_MAX;
  GK_CUDA(cudaStreamSynchronize(h->stream));
  return GK_OK;
}

int gk_core_level_add(gk_handle* h, int32_t level, int64_t n_fit, int64_t n_level_rows, const int32_t* rows,
                      const int32_t* cols, double* xdiag, double* ydiag, gk_stats* stats) {
  if (!h) return fail(GK_ERR_ARG, "null handle");
  if (!h->core_sum) return fail(GK_ERR_STATE, "gk_core_level_add: no sum begun (gk_core_sum_begin)");
  if (h->feature_kind == FK_NONE) return fail(GK_ERR_STATE, "gk_core_level_add: run the base kernel's feature pass first");
  if (level < 0 || level >= h->core_level)
    return fail(GK_ERR_ARG, "gk_core_level_add: core levels must be added in strictly descending order");
  if (!GRAM_RULES[h->feature_kind].dev_out)
    return fail(GK_ERR_UNSUPPORTED, std::string("gk_core_level_add: ") + GRAM_RULES[h->feature_kind].name +
                                        " Gram has no device output");
  GramReq q;
  GK_TRY(gram_request(h, h->feature_kind, n_fit, 0, 0, -1, nullptr, GK_F64, 0, xdiag, ydiag, &q));
  if (q.k_rows != n_level_rows) return fail(GK_ERR_ARG, "gk_core_level_add: the level's K has another number of rows");
  if ((q.k_rows && !rows) || !cols) return fail(GK_ERR_ARG, "gk_core_level_add: null index map");
  // every index in range and none twice: the scatter adds without atomics, one thread per element of the sum
  std::vector<uint8_t> seen((size_t)std::max(h->wl_sum_rows, h->wl_sum_cols), 0);
  for (int64_t j = 0; j < q.k_rows; ++j) {
    if (rows[j] < 0 || rows[j] >= h->wl_sum_rows || seen[rows[j]]++)
      return fail(GK_ERR_ARG, "gk_core_level_add: row map out of range or repeated");
  }
  std::fill(seen.begin(), seen.end(), 0);
  for (int64_t c = 0; c < q.k_cols; ++c) {
    if (cols[c] < 0 || cols[c] >= h->wl_sum_cols || seen[cols[c]]++)
      return fail(GK_ERR_ARG, "gk_core_level_add: column map out of range or repeated");
  }
  GK_CUDA(cudaSetDevice(h->dev));
  const size_t elems = (size_t)q.k_rows * q.k_cols;
  GK_TRY(h->wl_lvl.ensure(std::max<size_t>(elems, 1) * 8));
  GK_TRY(h->core_map.ensure((size_t)(q.k_rows + q.k_cols) * 4));
  int* d_rows = h->core_map.as<int>();
  int* d_cols = d_rows + q.k_rows;
  if (q.k_rows) GK_CUDA(cudaMemcpyAsync(d_rows, rows, (size_t)q.k_rows * 4, cudaMemcpyHostToDevice, h->stream));
  GK_CUDA(cudaMemcpyAsync(d_cols, cols, (size_t)q.k_cols * 4, cudaMemcpyHostToDevice, h->stream));
  q.flags |= GK_OUT_DEVICE; q.dev_out = true; q.K_out = h->wl_lvl.p; q.ld = q.k_cols;
  GK_TRY(gram_route(h, q, stats));
  if (elems) {
    core_scatter_add_f64<<<(int)std::min<size_t>((elems + 255) / 256, (size_t)h->sm_count * 16), 256, 0, h->stream>>>(
        q.k_rows, q.k_cols, h->wl_lvl.as<double>(), d_rows, d_cols, h->wl_sum.as<double>(), h->wl_sum_cols);
    LAUNCH_CHECK(h);
  }
  h->core_level = level;
  h->wl_sum_levels += 1;
  GK_CUDA(cudaStreamSynchronize(h->stream));
  return GK_OK;
}

}  // extern "C"

// ---------------------------------------------------------------------------
// OddSth (odd_sth.cuh).  gk_odd_features builds every root's DAG and the identities of its nodes, repeating the
// identity pass with another seed while a collision is detected, then counts phi per (graph, identity), C per
// identity, the self similarities, and splits the counts into one NeighborhoodSubgraphPairwiseDistance-layout table per
// bit of C.  odd_ctl: [collision | identities | entries of plane b (32) | columns of plane b (32)] u64.
static NspdLevel odd_plane(gk_handle* h, int b) {
  char* p = h->odd_blk.as<char>() + h->odd_off[b];
  const long long cap = h->odd_cap[b], M = h->odd_M[b];
  NspdLevel L;
  L.keys = reinterpret_cast<unsigned long long*>(p);
  L.cnt = reinterpret_cast<unsigned*>(p + cap * 8);
  L.colcnt = reinterpret_cast<unsigned*>(p + cap * 12);
  L.diag = reinterpret_cast<unsigned long long*>(p + cap * 12 + ((M + 1) * 4 + 7) / 8 * 8);
  L.part = reinterpret_cast<unsigned*>(L.diag + std::max<long long>(h->N, 1));
  return L;
}

constexpr int ODD_CTL_WORDS = 2 + 32 + 32;
constexpr int ODD_MAX_ATTEMPTS = 8;

// Device views of the node records (S slots) and the per-identity arrays.
struct OddNodes {
  unsigned long long* key;
  int *lab, *gr, *cb, *nc, *slot, *fid;
  int *rep_of, *Cf, *colb;
};

static OddNodes odd_nodes(gk_handle* h) {
  const size_t S1 = (size_t)std::max<long long>(h->odd_S, 1);
  OddNodes o;
  o.key = h->odd_nodes.as<unsigned long long>();
  o.lab = reinterpret_cast<int*>(o.key + S1);
  o.gr = o.lab + S1; o.cb = o.gr + S1; o.nc = o.cb + S1; o.slot = o.nc + S1; o.fid = o.slot + S1;
  o.rep_of = h->odd_feat.as<int>();
  o.Cf = o.rep_of + S1; o.colb = o.Cf + S1;
  return o;
}

extern "C" {

int gk_selftest_odd_collision(gk_handle* h, int32_t attempts) {
  if (!h || attempts < 0) return fail(GK_ERR_ARG, "gk_selftest_odd_collision: bad argument");
  h->odd_degen = attempts;
  return GK_OK;
}

}  // extern "C"

// The feature pass of gk_odd_features (n_levels = 1, the packed labels) and gk_wl_odd_features (one label set per WL
// level, `ids` [n_levels][V] disjoint across levels): every level's DAGs take their own node and child slots, so the
// identities of different levels never meet and one table of (graph, identity) counts holds the sum over the levels.
static int odd_features_impl(gk_handle* h, int32_t depth, int n_levels, const int32_t* ids, const int32_t* rank,
                             gk_stats* stats) {
  const int64_t N = h->N, V = h->V, E = h->E;
  const int64_t launches0 = h->launches;
  features_begin(h);
  const std::vector<int>& gp = h->graph_ptr_host;
  std::vector<long long> base(2 * (N + 1), 0);
  long long* nbase = base.data();
  long long* ebase = nbase + N + 1;
  int max_n = 1;
  for (int64_t g = 0; g < N; ++g) {
    const long long n = gp[g + 1] - gp[g], m = h->graph_eptr_host[g + 1] - h->graph_eptr_host[g];
    max_n = std::max<int>(max_n, (int)n);
    nbase[g + 1] = nbase[g] + n * n;
    ebase[g + 1] = ebase[g] + n * m;
  }
  const char* who = n_levels > 1 ? "gk_wl_odd_features" : "gk_odd_features";
  if (max_n > ODD_MAX_N) return fail(GK_ERR_UNSUPPORTED, std::string(who) + ": a graph has more than 4096 vertices");
  // the slots of all levels together, checked before anything is sized
  const long long S_lv = nbase[N], T_lv = ebase[N];
  const long long S = S_lv * n_levels, T = T_lv * n_levels;
  if (S >= (1LL << 30) || T >= (1LL << 30))
    return fail(GK_ERR_UNSUPPORTED, std::string(who) + ": 2^30 or more (root, vertex) or (root, edge) pairs" +
                                         (n_levels > 1 ? " over all WL levels" : ""));
  h->odd_S = S; h->odd_T = T; h->odd_maxC = 0;
  const size_t S1 = (size_t)std::max<long long>(S, 1), T1 = (size_t)std::max<long long>(T, 1);
  const size_t cap = std::max<size_t>(next_pow2(S1 * 2), 1024);
  const size_t LV = (size_t)n_levels * (size_t)V;
  GK_TRY(h->odd_aux.ensure(base.size() * 8 + std::max<size_t>(LV, 1) * 4 * (ids ? 2 : 1)));
  GK_TRY(h->odd_nodes.ensure(S1 * 32));
  GK_TRY(h->odd_ch.ensure(T1 * 4));
  GK_TRY(h->odd_tab.ensure(cap * 16));  // keys | representative | identity of the slot
  GK_TRY(h->odd_feat.ensure(S1 * 12));
  GK_TRY(h->odd_phi.ensure(cap * 12));
  GK_TRY(h->odd_ctl.ensure(ODD_CTL_WORDS * 8));
  GK_TRY(h->odd_diag.ensure((size_t)N * 8));
  GK_CUDA(cudaMemcpyAsync(h->odd_aux.p, base.data(), base.size() * 8, cudaMemcpyHostToDevice, h->stream));
  int* d_rank = reinterpret_cast<int*>(h->odd_aux.as<long long>() + base.size());
  int* d_ids = ids ? d_rank + std::max<size_t>(LV, 1) : h->labels0.as<int>();
  if (LV) GK_CUDA(cudaMemcpyAsync(d_rank, rank, LV * 4, cudaMemcpyHostToDevice, h->stream));
  if (LV && ids) GK_CUDA(cudaMemcpyAsync(d_ids, ids, LV * 4, cudaMemcpyHostToDevice, h->stream));
  const OddNodes o = odd_nodes(h);
  unsigned long long* tab = h->odd_tab.as<unsigned long long>();
  int* rep = reinterpret_cast<int*>(tab + cap);
  int* colid = rep + cap;
  unsigned long long* ctl = h->odd_ctl.as<unsigned long long>();
  unsigned long long* phi_keys = h->odd_phi.as<unsigned long long>();
  unsigned* phi_cnt = reinterpret_cast<unsigned*>(phi_keys + cap);
  GK_CUDA(cudaEventRecord(h->tev[2], h->stream));

  // ---- DAGs and identities; repeated with another seed while a collision is detected
  OddParams p;
  p.N = (int)N; p.V = V;
  p.n_levels = n_levels; p.S = S_lv; p.T = T_lv;
  p.graph_ptr = h->graph_ptr.as<int>(); p.row_ptr = h->row_ptr.as<int>(); p.col_idx = h->col_idx.as<int>();
  p.vgraph = h->vgraph.as<int>(); p.labels = d_ids; p.rank = d_rank;
  p.node_base = h->odd_aux.as<long long>(); p.edge_base = p.node_base + N + 1;
  p.depth = depth < 0 ? -1 : depth;
  p.n_pad = (max_n + 3) / 4 * 4;
  p.key = o.key; p.lab = o.lab; p.gr = o.gr; p.cb = o.cb; p.nc = o.nc; p.ch = h->odd_ch.as<int>();
  const size_t warp_smem = (size_t)p.n_pad * ODD_SMEM_PER_V;
  const int wpc = (int)std::max<size_t>(1, std::min<size_t>(ODD_MAX_WARPS, ((size_t)200 << 10) / warp_smem));
  const size_t smem = warp_smem * wpc;
  if (smem > (48 << 10))
    GK_CUDA(cudaFuncSetAttribute(odd_dags, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(cdiv(std::max<int64_t>((int64_t)LV, 1), wpc), (int64_t)h->sm_count * 16));
  int64_t retries = 0;
  for (int attempt = 0;; ++attempt) {
    if (attempt == ODD_MAX_ATTEMPTS)
      return fail(GK_ERR_STATE, std::string(who) + ": identity hashes collided on every attempt");
    p.seed = mix64(0x6f6464ULL + (unsigned long long)attempt * 0x9e3779b97f4a7c15ULL);
    p.degenerate = h->odd_degen > 0 ? 1 : 0;
    if (h->odd_degen > 0) h->odd_degen--;
    GK_CUDA(cudaMemsetAsync(ctl, 0, 8, h->stream));
    if (V) {
      odd_dags<<<grid, wpc * 32, smem, h->stream>>>(p);
      LAUNCH_CHECK(h);
    }
    GK_CUDA(cudaMemsetAsync(tab, 0xFF, cap * 8, h->stream));
    GK_CUDA(cudaMemsetAsync(rep, 0x7F, cap * 4, h->stream));
    if (S) {
      odd_insert<<<cdiv(S, 256), 256, 0, h->stream>>>(S, o.key, o.lab, tab, rep, cap - 1, o.slot);
      LAUNCH_CHECK(h);
      odd_verify<<<cdiv(S, 256), 256, 0, h->stream>>>(S, o.lab, o.nc, o.cb, h->odd_ch.as<int>(), o.slot, rep,
                                                       reinterpret_cast<unsigned*>(ctl));
      LAUNCH_CHECK(h);
    }
    unsigned long long coll = 0;
    GK_CUDA(cudaMemcpyAsync(&coll, ctl, 8, cudaMemcpyDeviceToHost, h->stream));
    GK_CUDA(cudaStreamSynchronize(h->stream));
    if (!coll) break;
    ++retries;
  }
  GK_CUDA(cudaEventRecord(h->tev[6], h->stream));

  // ---- identities numbered, C, phi, self similarities, entries per bit plane
  GK_CUDA(cudaMemsetAsync(ctl, 0, ODD_CTL_WORDS * 8, h->stream));
  GK_CUDA(cudaMemsetAsync(o.Cf, 0, S1 * 4, h->stream));
  GK_CUDA(cudaMemsetAsync(phi_keys, 0xFF, cap * 8, h->stream));
  GK_CUDA(cudaMemsetAsync(phi_cnt, 0, cap * 4, h->stream));
  GK_CUDA(cudaMemsetAsync(h->odd_diag.p, 0, (size_t)N * 8, h->stream));
  if (S) {
    odd_number<<<cdiv(S, 256), 256, 0, h->stream>>>(S, o.lab, o.slot, rep, colid, o.rep_of, ctl + 1);
    LAUNCH_CHECK(h);
    odd_count<<<cdiv(S, 256), 256, 0, h->stream>>>(S, o.lab, o.gr, o.slot, colid, o.rep_of, o.fid,
                                                   reinterpret_cast<unsigned*>(o.Cf), phi_keys, phi_cnt, cap - 1);
    LAUNCH_CHECK(h);
    odd_phi_stats<<<cdiv((long long)cap, 256), 256, 0, h->stream>>>(cap, phi_keys, phi_cnt,
                                                                    reinterpret_cast<unsigned*>(o.Cf),
                                                                    h->odd_diag.as<unsigned long long>(), ctl + 2);
    LAUNCH_CHECK(h);
  }
  std::vector<unsigned long long> hc(ODD_CTL_WORDS);
  GK_CUDA(cudaMemcpyAsync(hc.data(), ctl, ODD_CTL_WORDS * 8, cudaMemcpyDeviceToHost, h->stream));
  GK_CUDA(cudaStreamSynchronize(h->stream));
  const long long F = (long long)hc[1];
  h->odd_F = F;
  int B = 0;
  for (int b = 0; b < 32; ++b)
    if (hc[2 + b]) B = b + 1;
  h->odd_off.assign(B, 0); h->odd_cap.assign(B, 0); h->odd_M.assign(B, 0); h->odd_cols.assign(B, 0);
  size_t blk = 0;
  for (int b = 0; b < B; ++b) {
    const long long M = (long long)hc[2 + b];
    h->odd_M[b] = M;
    h->odd_cap[b] = (long long)std::max<size_t>(next_pow2((size_t)std::max<long long>(M, 1) * 2), 1024);
    h->odd_off[b] = (long long)blk;
    blk += nspd_level_bytes(h->odd_cap[b], M, N);
  }
  GK_TRY(h->odd_blk.ensure(std::max<size_t>(blk, 256)));
  if (blk) GK_CUDA(cudaMemsetAsync(h->odd_blk.p, 0, blk, h->stream));
  for (int b = 0; b < B; ++b) {
    const NspdLevel L = odd_plane(h, b);
    const size_t pcap = (size_t)h->odd_cap[b];
    GK_CUDA(cudaMemsetAsync(L.keys, 0xFF, pcap * 8, h->stream));
    if (!h->odd_M[b]) continue;
    odd_plane_cols<<<cdiv(F, 256), 256, 0, h->stream>>>((int)F, reinterpret_cast<unsigned*>(o.Cf), b, o.colb, ctl + 34 + b);
    LAUNCH_CHECK(h);
    odd_plane_fill<<<cdiv((long long)cap, 256), 256, 0, h->stream>>>(cap, phi_keys, phi_cnt, reinterpret_cast<unsigned*>(o.Cf),
                                                                     b, o.colb, L.keys, L.cnt, pcap - 1);
    LAUNCH_CHECK(h);
    nspd_level_stats<<<cdiv((long long)pcap, 256), 256, 0, h->stream>>>(pcap, L.keys, L.cnt, L.colcnt, L.diag, L.part);
    LAUNCH_CHECK(h);
  }
  GK_CUDA(cudaEventRecord(h->tev[3], h->stream));
  GK_CUDA(cudaMemcpyAsync(hc.data() + 34, ctl + 34, 32 * 8, cudaMemcpyDeviceToHost, h->stream));
  GK_CUDA(cudaStreamSynchronize(h->stream));
  for (int b = 0; b < B; ++b) h->odd_cols[b] = (long long)hc[34 + b];
  h->n_columns = F;
  features_publish(h, FK_ODD);
  if (stats) {
    memset(stats, 0, sizeof(*stats));
    stats->n_graphs = N; stats->n_vertices = V; stats->n_edges = E;
    stats->n_levels = B;
    for (int b = 0; b < B; ++b) stats->level_dims[b] = h->odd_cols[b];
    stats->n_columns = F;
    stats->n_entries = S;
    stats->hash_retries = retries;
    stats->kernel_launches = h->launches - launches0;
    stats->ms_features = ev_ms(h->tev[2], h->tev[3]);
    stats->ms_hash = ev_ms(h->tev[2], h->tev[6]);
    stats->ms_columns = ev_ms(h->tev[6], h->tev[3]);
  }
  return GK_OK;
}

extern "C" {

int gk_odd_features(gk_handle* h, int32_t depth, const int32_t* rank, int32_t flags, gk_stats* stats) {
  GK_TRY(need_packed(h, "gk_odd_features"));
  if (!h->has_labels) return fail(GK_ERR_ARG, "gk_odd_features: vertex labels are required");
  if (depth == 0) return fail(GK_ERR_ARG, "gk_odd_features: h must be > 0 (or < 0 for no limit)");
  if (flags != 0) return fail(GK_ERR_ARG, "gk_odd_features: no flags are defined");
  if (!rank && h->V) return fail(GK_ERR_ARG, "gk_odd_features: null rank table");
  return odd_features_impl(h, depth, 1, nullptr, rank, stats);
}

int gk_wl_odd_features(gk_handle* h, int32_t depth, int32_t n_iter, const int32_t* ids, const int32_t* rank,
                       int32_t flags, gk_stats* stats) {
  GK_TRY(need_packed(h, "gk_wl_odd_features"));
  if (depth == 0) return fail(GK_ERR_ARG, "gk_wl_odd_features: h must be > 0 (or < 0 for no limit)");
  if (n_iter < 0 || n_iter >= MAX_LEVELS) return fail(GK_ERR_ARG, "gk_wl_odd_features: n_iter out of range");
  if (flags != 0) return fail(GK_ERR_ARG, "gk_wl_odd_features: no flags are defined");
  if ((!ids || !rank) && h->V) return fail(GK_ERR_ARG, "gk_wl_odd_features: null label or rank table");
  // label ids are hashed and compared, ranks ordered as u32: both must be non-negative, and a level's ids must not
  // reach into another level's (the host makes them disjoint by offsetting each level past the previous one)
  const int64_t V = h->V;
  int prev_hi = -1;
  for (int lv = 0; lv <= n_iter; ++lv) {
    int lo = INT_MAX, hi = -1;
    for (int64_t v = 0; v < V; ++v) {
      const int32_t a = ids[(size_t)lv * V + v];
      if (a < 0 || rank[(size_t)lv * V + v] < 0) return fail(GK_ERR_ARG, "gk_wl_odd_features: negative label id or rank");
      lo = std::min<int>(lo, a); hi = std::max<int>(hi, a);
    }
    if (V && lo <= prev_hi) return fail(GK_ERR_ARG, "gk_wl_odd_features: label ids of two levels overlap");
    prev_hi = hi;
  }
  return odd_features_impl(h, depth, n_iter + 1, ids, rank, stats);
}

}  // extern "C"

// The signature of every identity, from its representative node: label id, children's identities in order, C.
static int odd_host_signatures(gk_handle* h, std::vector<int>* label, std::vector<int64_t>* off, std::vector<int>* child,
                               std::vector<int>* C) {
  if (h->feature_kind != FK_ODD) return fail(GK_ERR_STATE, "gk_odd_signatures: run gk_odd_features first");
  GK_CUDA(cudaSetDevice(h->dev));
  const long long S = h->odd_S, T = h->odd_T, F = h->odd_F;
  const OddNodes o = odd_nodes(h);
  std::vector<int> lab(S), cb(S), nc(S), fid(S), ch(T), rep_of(F);
  C->resize(F);
  GK_CUDA(cudaStreamSynchronize(h->stream));
  if (S) {
    GK_CUDA(cudaMemcpy(lab.data(), o.lab, S * 4, cudaMemcpyDeviceToHost));
    GK_CUDA(cudaMemcpy(cb.data(), o.cb, S * 4, cudaMemcpyDeviceToHost));
    GK_CUDA(cudaMemcpy(nc.data(), o.nc, S * 4, cudaMemcpyDeviceToHost));
    GK_CUDA(cudaMemcpy(fid.data(), o.fid, S * 4, cudaMemcpyDeviceToHost));
  }
  if (T) GK_CUDA(cudaMemcpy(ch.data(), h->odd_ch.p, T * 4, cudaMemcpyDeviceToHost));
  if (F) {
    GK_CUDA(cudaMemcpy(rep_of.data(), o.rep_of, F * 4, cudaMemcpyDeviceToHost));
    GK_CUDA(cudaMemcpy(C->data(), o.Cf, F * 4, cudaMemcpyDeviceToHost));
  }
  label->resize(F);
  off->assign(F + 1, 0);
  child->clear();
  for (long long f = 0; f < F; ++f) {
    const int r = rep_of[f];
    (*label)[f] = lab[r];
    for (int k = 0; k < nc[r]; ++k) child->push_back(fid[ch[cb[r] + k]]);
    (*off)[f + 1] = (int64_t)child->size();
  }
  return GK_OK;
}

extern "C" {

int gk_odd_info(gk_handle* h, int64_t* info3) {
  if (!h || !info3) return fail(GK_ERR_ARG, "gk_odd_info: null argument");
  std::vector<int> label, child, C;
  std::vector<int64_t> off;
  GK_TRY(odd_host_signatures(h, &label, &off, &child, &C));
  info3[0] = (int64_t)label.size();
  info3[1] = (int64_t)child.size();
  info3[2] = C.empty() ? 0 : *std::max_element(C.begin(), C.end());
  return GK_OK;
}

int gk_odd_signatures(gk_handle* h, int32_t* label, int64_t* child_off, int32_t* child, int32_t* C) {
  if (!h || !label || !child_off || !C) return fail(GK_ERR_ARG, "gk_odd_signatures: null argument");
  std::vector<int> lb, ch, c;
  std::vector<int64_t> off;
  GK_TRY(odd_host_signatures(h, &lb, &off, &ch, &c));
  if (!lb.empty()) {
    memcpy(label, lb.data(), lb.size() * 4);
    memcpy(C, c.data(), c.size() * 4);
  }
  memcpy(child_off, off.data(), off.size() * 8);
  if (!ch.empty()) {
    if (!child) return fail(GK_ERR_ARG, "gk_odd_signatures: null child array");
    memcpy(child, ch.data(), ch.size() * 4);
  }
  return GK_OK;
}

}  // extern "C"

// Gram of OddSth (gram_path 14): per bit plane b of C, the exact integer Gram G_b of its count table as fp64 counts,
// folded into K as 2^b G_b (one count matrix live), so K = sum_f C[f] phi_i[f] phi_j[f] exactly below 2^53.  The self
// similarities d (sum_f C[f] phi[f]^2, u64 from the feature pass) give GK_NORMALIZE's K / sqrt(d_i d_j) and xdiag /
// ydiag.  Rows go in chunks when one plane's count matrix of the whole request would exceed 8 GiB
// (GRAKEL_B200_ODD_C_BUDGET=<bytes> lowers it).
static int gram_odd(gk_handle* h, const GramReq& q, gk_stats* stats) {
  const int64_t N = h->N, n_fit = q.n_fit, k_rows = q.k_rows, k_cols = q.k_cols;
  const int B = (int)h->odd_M.size();
  const int64_t launches0 = h->launches;
  F64Out out;
  GK_TRY(f64_target(h, q, &out));
  const int64_t ldc = (k_cols + 7) / 8 * 8;
  size_t c_budget = (size_t)8 << 30;
  if (const char* e = getenv("GRAKEL_B200_ODD_C_BUDGET")) c_budget = std::max<size_t>(1, strtoull(e, nullptr, 10));
  const int64_t chunk = std::max<int64_t>(1, std::min<int64_t>(std::max<int64_t>(k_rows, 1), (int64_t)(c_budget / ((size_t)ldc * 8))));
  GK_TRY(h->nh_C.ensure((size_t)chunk * ldc * 8));
  double* C = h->nh_C.as<double>();
  const int32_t gflags = (q.flags & (GK_GRAM_SIMT | GK_DENSE_ALL)) | GK_FULL_TILES | GK_OUT_DEVICE;
  std::vector<float> ms_plane(64, 0.f);
  float ms_fold = 0.f;
  int64_t max_T = 0, gram_launches = 0, elem_bytes = 0, max_count = 0;
  for (int64_t cb = q.row_begin; cb < q.row_end; cb += chunk) {
    const int64_t ce = std::min<int64_t>(q.row_end, cb + chunk), rows = ce - cb;
    double* o = out.p + (size_t)(cb - q.row_begin) * out.ld;
    GK_CUDA(cudaMemset2DAsync(o, (size_t)out.ld * 8, 0, (size_t)k_cols * 8, (size_t)rows, h->stream));
    for (int b = 0; b < B; ++b) {
      if (!h->odd_M[b]) continue;
      const NspdLevel L = odd_plane(h, b);
      IntBlock fb;
      fb.keys = L.keys; fb.cnt = L.cnt; fb.cap = (size_t)h->odd_cap[b];
      fb.colcnt = L.colcnt; fb.col_cap = h->odd_M[b] + 1; fb.n_columns = h->odd_cols[b];
      fb.diag = L.diag; fb.part_max = L.part; fb.part_new = L.part + 1; fb.n_part = 1;
      fb.prologue_on_host = false;
      GramReq lq;
      GK_TRY(gram_request(h, FK_WL, n_fit, gflags, cb, ce, C, GK_F64, ldc, nullptr, nullptr, &lq));
      gk_stats st;
      memset(&st, 0, sizeof(st));
      GK_TRY(gram_int(h, lq, fb, &st));
      ms_plane[b] += st.ms_total;
      max_T = std::max<int64_t>(max_T, st.threshold);
      max_count = std::max<int64_t>(max_count, st.max_count);
      gram_launches += st.gemm_launches;
      elem_bytes = std::max<int64_t>(elem_bytes, st.gemm_elem_bytes);
      if (rows > 0) {
        GK_CUDA(cudaEventRecord(h->tev[0], h->stream));
        odd_fold<<<cdiv(rows * k_cols, 256), 256, 0, h->stream>>>((int)rows, (int)k_cols, C, ldc, b, o, out.ld);
        LAUNCH_CHECK(h);
        GK_CUDA(cudaEventRecord(h->tev[1], h->stream));
        GK_CUDA(cudaEventSynchronize(h->tev[1]));
        ms_fold += ev_ms(h->tev[0], h->tev[1]);
      }
    }
  }
  // gram_int left its planes' self similarities in diag_f64: replace them with d
  GK_TRY(h->diag_f64.ensure((size_t)N * 8));
  odd_diag_f64<<<cdiv(N, 256), 256, 0, h->stream>>>((int)N, h->odd_diag.as<unsigned long long>(), h->diag_f64.as<double>());
  LAUNCH_CHECK(h);
  GK_TRY(f64_deliver(h, q, out, true, h->ev[14], h->ev[15]));
  if (stats) {
    stats->n_graphs = N; stats->n_vertices = h->V; stats->n_edges = h->E;
    stats->n_levels = B;
    stats->gram_path = 14;
    stats->threshold = max_T;
    stats->max_count = max_count;
    stats->gemm_launches = gram_launches + (h->launches - launches0);
    stats->gemm_elem_bytes = elem_bytes;
    float tot = ms_fold;
    for (int b = 0; b < B && b < 64; ++b) { stats->ms_level_gram[b] = ms_plane[b]; tot += ms_plane[b]; }
    stats->ms_gemm = tot - ms_fold;
    stats->ms_combine = ms_fold;
    stats->ms_d2h = ev_ms(h->ev[14], h->ev[15]);
    stats->ms_total = tot + stats->ms_d2h;
  }
  return GK_OK;
}

// ---------------------------------------------------------------------------
// MultiscaleLaplacian (multiscale_laplacian.cuh).  A staged pipeline, because the reference's eigen-decompositions
// of the sampled blocks run on the host between the levels:
//   gk_ml_begin    dense adjacency, radius-l balls and the attributes of the packed block (the level-0 features)
//   gk_ml_project  U <- U Q (phi ksi at level 0, K_proj Q after each level)
//   gk_ml_level    every vertex's record at level l, the projection block against the level's sample records
//   gk_ml_finish   every graph's final record, appended to the fitted graphs' records for gk_gram (gram_path 15)
static int ml_check_err(gk_handle* h) {
  unsigned err = 0;
  GK_CUDA(cudaMemcpyAsync(&err, h->ml_ctl.p, 4, cudaMemcpyDeviceToHost, h->stream));
  GK_CUDA(cudaStreamSynchronize(h->stream));
  if (err & 2u) return fail(GK_ERR_UNSUPPORTED, "MultiscaleLaplacian: a non-symmetric adjacency matrix");
  if (err & 1u) return fail(GK_ERR_RANGE, "MultiscaleLaplacian: a Cholesky factorisation met a non-positive pivot");
  return GK_OK;
}

static size_t ml_unit_smem(int mcap, int P) {
  return ((size_t)std::max(mcap * mcap, P * P) + (size_t)mcap * P + (size_t)P * P) * 8;
}

// Records of n_units units (vertices with `ball`, else graphs) from the current features, into `rec`.
static int ml_records(gk_handle* h, const unsigned long long* ball, int dup_loops, int mcap, int n_units, double* rec) {
  if (n_units <= 0) return GK_OK;
  MlUnits p;
  p.graph_ptr = h->graph_ptr.as<int>(); p.vgraph = h->vgraph.as<int>();
  p.adj_off = h->ml_adj_off.as<long long>(); p.adj = h->ml_adj.as<double>();
  p.ball = ball; p.dup_loops = dup_loops;
  p.U = h->ml_U.as<double>(); p.P = h->ml_w;
  p.gamma = h->ml_gamma; p.heta = h->ml_heta;
  p.n_units = n_units; p.rec = rec;
  p.err = h->ml_ctl.as<unsigned>();
  const size_t smem = ml_unit_smem(mcap, h->ml_w);
  GK_CUDA(cudaFuncSetAttribute(ml_vertex_C, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int per_sm = 0;
  GK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, ml_vertex_C, ML_THREADS, smem));
  const int grid = (int)std::min<long long>(n_units, (long long)h->sm_count * std::max(per_sm, 1));
  ml_vertex_C<<<grid, ML_THREADS, smem, h->stream>>>(p, mcap);
  LAUNCH_CHECK(h);
  return GK_OK;
}

static int ml_flg_grid(gk_handle* h, const void* fn, int P, long long n_pairs, size_t* smem, int* grid) {
  *smem = (size_t)ML_FLG_WARPS * P * P * 8;
  GK_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max<size_t>(*smem, 1)));
  int per_sm = 0;
  GK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, 32 * ML_FLG_WARPS, *smem));
  *grid = (int)std::max<long long>(1, std::min<long long>((n_pairs + ML_FLG_WARPS - 1) / ML_FLG_WARPS,
                                                           (long long)h->sm_count * std::max(per_sm, 1)));
  return GK_OK;
}

static int ml_ready(gk_handle* h, const char* who) {
  if (!h) return fail(GK_ERR_ARG, "null handle");
  if (h->ml_L < 0 || !h->ml_U.p || h->ml_w <= 0) return fail(GK_ERR_STATE, std::string(who) + ": call gk_ml_begin first");
  return GK_OK;
}

extern "C" {

int gk_ml_begin(gk_handle* h, int32_t L, double gamma, double heta, const double* phi, int32_t dim, gk_stats* stats) {
  GK_TRY(need_packed(h, "gk_ml_begin"));
  if (L < 0 || L > 64) return fail(GK_ERR_UNSUPPORTED, "gk_ml_begin: L outside [0, 64]");
  if (!(gamma > 0.0) || !(heta > 0.0) || !std::isfinite(gamma) || !std::isfinite(heta))
    return fail(GK_ERR_UNSUPPORTED, "gk_ml_begin: gamma and heta must be positive and finite (the Cholesky route)");
  if (dim < 1 || !phi) return fail(GK_ERR_ARG, "gk_ml_begin: no attributes");
  if (h->max_graph_size > ML_NMAX)
    return fail(GK_ERR_UNSUPPORTED, "gk_ml_begin: a graph of more than 128 vertices (the neighbourhood matrix lives in "
                                    "shared memory)");
  const int64_t N = h->N, V = h->V;
  std::vector<long long> off(N + 1, 0);
  for (int64_t g = 0; g < N; ++g) {
    const long long n = h->graph_ptr_host[g + 1] - h->graph_ptr_host[g];
    off[g + 1] = off[g] + n * n;
  }
  features_begin(h);
  h->ml_w = 0;  // no session until this call completes
  GK_CUDA(cudaEventRecord(h->tev[0], h->stream));
  GK_TRY(h->ml_adj_off.ensure((N + 1) * 8));
  GK_TRY(h->ml_adj.ensure(std::max<long long>(off[N], 1) * 8));
  GK_TRY(h->ml_ball.ensure(std::max<long long>((long long)L * V * 2, 1) * 8));
  GK_TRY(h->ml_U.ensure(std::max<long long>(V * dim, 1) * 8));
  GK_TRY(h->ml_ctl.ensure(16));
  GK_CUDA(cudaMemcpyAsync(h->ml_adj_off.p, off.data(), (N + 1) * 8, cudaMemcpyHostToDevice, h->stream));
  GK_CUDA(cudaMemcpyAsync(h->ml_U.p, phi, (size_t)V * dim * 8, cudaMemcpyHostToDevice, h->stream));
  GK_CUDA(cudaMemsetAsync(h->ml_adj.p, 0, std::max<long long>(off[N], 1) * 8, h->stream));
  GK_CUDA(cudaMemsetAsync(h->ml_ctl.p, 0, 16, h->stream));
  GK_CUDA(cudaEventRecord(h->tev[1], h->stream));
  unsigned long long* ball = h->ml_ball.as<unsigned long long>();
  std::vector<int> mcap(L + 1, 1);
  if (V > 0) {
    const int grid = cdiv(V, 256);
    ml_dense_adj<<<grid, 256, 0, h->stream>>>((int)V, h->graph_ptr.as<int>(), h->vgraph.as<int>(), h->row_ptr.as<int>(),
                                             h->col_idx.as<int>(), h->has_weights ? h->weights.as<double>() : nullptr,
                                             h->ml_adj_off.as<long long>(), h->ml_adj.as<double>());
    LAUNCH_CHECK(h);
    if (L >= 1) {
      ml_ball1<<<grid, 256, 0, h->stream>>>((int)V, h->graph_ptr.as<int>(), h->vgraph.as<int>(),
                                            h->ml_adj_off.as<long long>(), h->ml_adj.as<double>(), ball,
                                            h->ml_ctl.as<unsigned>());
      LAUNCH_CHECK(h);
    }
    for (int l = 2; l <= L; ++l) {
      ml_ball_next<<<grid, 256, 0, h->stream>>>((int)V, h->graph_ptr.as<int>(), h->vgraph.as<int>(),
                                                ball + (size_t)(l - 2) * V * 2, ball + (size_t)(l - 1) * V * 2);
      LAUNCH_CHECK(h);
    }
  }
  GK_CUDA(cudaEventRecord(h->tev[2], h->stream));
  // the symmetry check, and the largest neighbourhood of every level (it sizes the record kernel's shared memory)
  if (L >= 1 && V > 0) {
    std::vector<unsigned long long> hb((size_t)L * V * 2);
    GK_CUDA(cudaMemcpyAsync(hb.data(), ball, hb.size() * 8, cudaMemcpyDeviceToHost, h->stream));
    GK_TRY(ml_check_err(h));
    for (int l = 1; l <= L; ++l) {
      int mx = 1;
      for (int64_t u = 0; u < V; ++u) {
        const unsigned long long* b = &hb[((size_t)(l - 1) * V + u) * 2];
        mx = std::max(mx, __builtin_popcountll(b[0]) + __builtin_popcountll(b[1]));
      }
      mcap[l] = std::min(ML_MMAX, mx + (l == 1 ? 1 : 0));  // + a self-loop's second listing
    }
  } else {
    GK_TRY(ml_check_err(h));
  }
  h->ml_L = L; h->ml_w = dim;
  for (int l = 0; l <= L; ++l) h->ml_mcap[l] = mcap[l];
  h->ml_gamma = gamma; h->ml_heta = heta;
  h->ml_nrec = 0;
  if (stats) {
    stats->n_graphs = N; stats->n_vertices = h->V; stats->n_edges = h->E;
    stats->n_levels = L;
    stats->ms_h2d = ev_ms(h->tev[0], h->tev[1]);
    stats->ms_features = ev_ms(h->tev[1], h->tev[2]);
  }
  return GK_OK;
}

int gk_ml_project(gk_handle* h, const double* Q, int32_t rows, int32_t cols, gk_stats* stats) {
  GK_TRY(ml_ready(h, "gk_ml_project"));
  if (!Q || rows != h->ml_w) return fail(GK_ERR_ARG, "gk_ml_project: Q must have as many rows as the features have columns");
  if (cols < 1 || cols > ML_PMAX)
    return fail(GK_ERR_UNSUPPORTED, "gk_ml_project: the feature width must lie in [1, 32] (got " + std::to_string(cols) + ")");
  GK_CUDA(cudaSetDevice(h->dev));
  const long long V = h->V;
  GK_TRY(h->ml_aux.ensure((size_t)rows * cols * 8));
  GK_TRY(h->ml_U2.ensure(std::max<long long>(V * cols, 1) * 8));
  GK_CUDA(cudaMemcpyAsync(h->ml_aux.p, Q, (size_t)rows * cols * 8, cudaMemcpyHostToDevice, h->stream));
  GK_CUDA(cudaEventRecord(h->tev[0], h->stream));
  if (V > 0) {
    ml_matmul<<<(int)std::min<long long>(cdiv(V * cols, 256), (long long)h->sm_count * 16), 256, 0, h->stream>>>(
        V, rows, cols, h->ml_U.as<double>(), h->ml_aux.as<double>(), h->ml_U2.as<double>());
    LAUNCH_CHECK(h);
  }
  GK_CUDA(cudaEventRecord(h->tev[1], h->stream));
  GK_CUDA(cudaStreamSynchronize(h->stream));
  std::swap(h->ml_U, h->ml_U2);
  h->ml_w = cols;
  if (stats) stats->ms_combine = ev_ms(h->tev[0], h->tev[1]);
  return GK_OK;
}

int gk_ml_level(gk_handle* h, int32_t level, const int32_t* samples, int32_t ns, const double* samp_rec,
                double* samp_rec_out, double* K_samples, gk_stats* stats) {
  GK_TRY(ml_ready(h, "gk_ml_level"));
  if (level < 1 || level > h->ml_L) return fail(GK_ERR_ARG, "gk_ml_level: level outside [1, L]");
  if (ns < 1) return fail(GK_ERR_ARG, "gk_ml_level: no samples");
  if (ns > ML_NSMAX) return fail(GK_ERR_UNSUPPORTED, "gk_ml_level: more than 1024 samples");
  if (!samples == !samp_rec) return fail(GK_ERR_ARG, "gk_ml_level: give either sample ids or sample records");
  if (h->ml_w > ML_PMAX) return fail(GK_ERR_UNSUPPORTED, "gk_ml_level: records of more than 32 features");
  GK_CUDA(cudaSetDevice(h->dev));
  const long long V = h->V, P = h->ml_w, stride = P * P + 1;
  GK_TRY(h->ml_vrec.ensure(std::max<long long>(V * stride, 1) * 8));
  GK_TRY(h->ml_samp.ensure((size_t)ns * stride * 8));
  GK_TRY(h->ml_U2.ensure(std::max<long long>(V * ns, 1) * 8));
  GK_TRY(h->ml_aux.ensure((size_t)ns * 4 + (size_t)ns * ns * 8 + 64));
  int* d_ids = h->ml_aux.as<int>();
  double* d_kss = reinterpret_cast<double*>(h->ml_aux.as<char>() + ((size_t)ns * 4 + 63) / 64 * 64);
  if (samples) {
    for (int i = 0; i < ns; ++i)
      if (samples[i] < 0 || samples[i] >= V) return fail(GK_ERR_ARG, "gk_ml_level: sample id out of range");
    GK_CUDA(cudaMemcpyAsync(d_ids, samples, (size_t)ns * 4, cudaMemcpyHostToDevice, h->stream));
  } else {
    GK_CUDA(cudaMemcpyAsync(h->ml_samp.p, samp_rec, (size_t)ns * stride * 8, cudaMemcpyHostToDevice, h->stream));
  }
  GK_CUDA(cudaMemsetAsync(h->ml_ctl.p, 0, 4, h->stream));
  GK_CUDA(cudaEventRecord(h->tev[0], h->stream));
  GK_TRY(ml_records(h, h->ml_ball.as<unsigned long long>() + (size_t)(level - 1) * V * 2, level == 1 ? 1 : 0,
                    h->ml_mcap[level], (int)V, h->ml_vrec.as<double>()));
  if (samples && ns > 0) {
    ml_gather_rows<<<cdiv((long long)ns * stride, 256), 256, 0, h->stream>>>(ns, d_ids, h->ml_vrec.as<double>(), stride,
                                                                           h->ml_samp.as<double>());
    LAUNCH_CHECK(h);
  }
  GK_CUDA(cudaEventRecord(h->tev[1], h->stream));
  if (V > 0) {
    size_t smem;
    int grid;
    GK_TRY(ml_flg_grid(h, (const void*)ml_flg_project, (int)P, V * ns, &smem, &grid));
    ml_flg_project<<<grid, 32 * ML_FLG_WARPS, smem, h->stream>>>(h->ml_samp.as<double>(), h->ml_vrec.as<double>(), (int)P,
                                                                 V, ns, h->ml_U2.as<double>(), h->ml_ctl.as<unsigned>());
    LAUNCH_CHECK(h);
  }
  GK_CUDA(cudaEventRecord(h->tev[2], h->stream));
  if (samples && K_samples) {
    ml_gather_rows<<<cdiv((long long)ns * ns, 256), 256, 0, h->stream>>>(ns, d_ids, h->ml_U2.as<double>(), ns, d_kss);
    LAUNCH_CHECK(h);
    GK_CUDA(cudaMemcpyAsync(K_samples, d_kss, (size_t)ns * ns * 8, cudaMemcpyDeviceToHost, h->stream));
  }
  if (samples && samp_rec_out)
    GK_CUDA(cudaMemcpyAsync(samp_rec_out, h->ml_samp.p, (size_t)ns * stride * 8, cudaMemcpyDeviceToHost, h->stream));
  GK_CUDA(cudaEventRecord(h->tev[3], h->stream));
  GK_TRY(ml_check_err(h));
  std::swap(h->ml_U, h->ml_U2);
  h->ml_w = ns;
  if (stats) {
    stats->n_graphs = h->N; stats->n_vertices = V;
    stats->ms_features = ev_ms(h->tev[0], h->tev[1]);
    stats->ms_rw = ev_ms(h->tev[1], h->tev[2]);
    stats->ms_d2h = ev_ms(h->tev[2], h->tev[3]);
  }
  return GK_OK;
}

int gk_ml_finish(gk_handle* h, const double* fit_rec, int64_t n_fit, double* rec_out, gk_stats* stats) {
  GK_TRY(ml_ready(h, "gk_ml_finish"));
  if (n_fit < 0 || (n_fit > 0 && !fit_rec)) return fail(GK_ERR_ARG, "gk_ml_finish: bad fitted records");
  if (h->ml_w > ML_PMAX) return fail(GK_ERR_UNSUPPORTED, "gk_ml_finish: records of more than 32 features");
  GK_CUDA(cudaSetDevice(h->dev));
  const long long N = h->N, P = h->ml_w, stride = P * P + 1;
  GK_TRY(h->ml_rec.ensure((size_t)(n_fit + N) * stride * 8));
  double* rec = h->ml_rec.as<double>();
  if (n_fit > 0) GK_CUDA(cudaMemcpyAsync(rec, fit_rec, (size_t)n_fit * stride * 8, cudaMemcpyHostToDevice, h->stream));
  GK_CUDA(cudaMemsetAsync(h->ml_ctl.p, 0, 4, h->stream));
  GK_CUDA(cudaEventRecord(h->tev[0], h->stream));
  GK_TRY(ml_records(h, nullptr, 0, std::max(h->max_graph_size, 1), (int)N, rec + (size_t)n_fit * stride));
  GK_CUDA(cudaEventRecord(h->tev[1], h->stream));
  if (rec_out)
    GK_CUDA(cudaMemcpyAsync(rec_out, rec + (size_t)n_fit * stride, (size_t)N * stride * 8, cudaMemcpyDeviceToHost, h->stream));
  GK_TRY(ml_check_err(h));
  h->ml_nrec = n_fit + N;
  features_publish(h, FK_ML);
  if (stats) stats->ms_features = ev_ms(h->tev[0], h->tev[1]);
  return GK_OK;
}

}  // extern "C"

// Gram of MultiscaleLaplacian (gram_path 15): K[r][c] = flg(record a0 + r, record c), one warp per pair; fp64, host
// or GK_OUT_DEVICE output, GK_NORMALIZE, n_fit and row ranges.  The self similarities come from the same pair
// function, so a square K's diagonal equals them bit for bit; the full square case computes the upper triangle and
// mirrors it.
static int gram_ml(gk_handle* h, const GramReq& q, gk_stats* stats) {
  const int64_t N = q.N, k_rows = q.k_rows, k_cols = q.k_cols;
  const int P = h->ml_w;
  const int64_t launches0 = h->launches;
  F64Out out;
  GK_TRY(f64_target(h, q, &out));
  GK_TRY(h->diag_f64.ensure((size_t)N * 8));
  GK_CUDA(cudaMemsetAsync(h->ml_ctl.p, 0, 4, h->stream));
  const double* rec = h->ml_rec.as<double>();
  unsigned* err = h->ml_ctl.as<unsigned>();
  GK_CUDA(cudaEventRecord(h->tev[2], h->stream));
  size_t smem;
  int grid;
  GK_TRY(ml_flg_grid(h, (const void*)ml_flg_gram, P, N, &smem, &grid));
  ml_flg_gram<<<grid, 32 * ML_FLG_WARPS, smem, h->stream>>>(rec, P, RW_PAIRS_DIAG, N, (int)N, (int)N, 0,
                                                            h->diag_f64.as<double>(), 1, err);
  LAUNCH_CHECK(h);
  const bool mirror = q.full_square && !(q.flags & GK_FULL_TILES);
  const long long n_pairs = mirror ? N * (N + 1) / 2 : k_rows * k_cols;
  if (n_pairs > 0) {
    GK_TRY(ml_flg_grid(h, (const void*)ml_flg_gram, P, n_pairs, &smem, &grid));
    ml_flg_gram<<<grid, 32 * ML_FLG_WARPS, smem, h->stream>>>(rec, P, mirror ? RW_PAIRS_TRIANGLE : RW_PAIRS_RECT, n_pairs,
                                                              (int)k_rows, (int)k_cols, q.a0, out.p, out.ld, err);
    LAUNCH_CHECK(h);
  }
  GK_CUDA(cudaEventRecord(h->tev[3], h->stream));
  GK_TRY(ml_check_err(h));
  GK_TRY(f64_deliver(h, q, out, true, h->tev[3], h->tev[4]));
  if (stats) {
    stats->n_graphs = N; stats->n_vertices = h->V; stats->n_edges = h->E;
    stats->gram_path = 15;
    stats->gemm_tiles = n_pairs;
    stats->gemm_launches = h->launches - launches0;
    stats->ms_rw = ev_ms(h->tev[2], h->tev[3]);
    stats->ms_gemm = stats->ms_rw;
    stats->ms_d2h = ev_ms(h->tev[3], h->tev[4]);
    stats->ms_total = stats->ms_rw + stats->ms_d2h;
  }
  return GK_OK;
}

// ---------------------------------------------------------------------------
// SvmTheta (svm_theta.cuh).  gk_svmt_solve launches the eigenvalue and SMO kernels and returns; the caller draws the
// samples on the host (gk_svmt_draw, which needs no alphas) while they run; gk_svmt_phi then forms phi and leaves the
// first level of every graph, after the fitted graphs' (n_fit), for gk_gram (gram_path 16).
// Gram of SvmTheta (gram_path 16): K[r][c] = phi0[a0 + r] phi0[c] (the reference's default metric np.inner(x, y)[0, 0])
// by the fp64 CUDA-core Gram over a one-column feature matrix, a single rounded product per entry; the self
// similarities are the same products, so GK_NORMALIZE divides by sqrt(d_r d_c) as numpy's K / sqrt(outer(d, d)).
static int gram_svmt(gk_handle* h, const GramReq& q, gk_stats* stats) {
  const int64_t N = q.N, k_rows = q.k_rows, k_cols = q.k_cols;
  const int64_t launches0 = h->launches;
  F64Out out;
  GK_TRY(f64_target(h, q, &out));
  GK_TRY(h->diag_f64.ensure((size_t)N * 8));
  const double* rec = h->svmt_rec.as<double>();
  GK_CUDA(cudaEventRecord(h->tev[2], h->stream));
  svmt_diag<<<(int)std::max<int64_t>(1, std::min<int64_t>(cdiv(N, 256), (int64_t)h->sm_count * 8)), 256, 0, h->stream>>>(
      rec, N, h->diag_f64.as<double>());
  LAUNCH_CHECK(h);
  if (k_rows > 0) {
    dim3 grid((unsigned)cdiv(k_cols, 64), (unsigned)cdiv(k_rows, 64));
    gram_f64_kernel<<<grid, 256, 0, h->stream>>>(rec, 1, q.a0, q.a1, 0, (int)q.n_fit, out.p, out.ld);
    LAUNCH_CHECK(h);
  }
  GK_CUDA(cudaEventRecord(h->tev[3], h->stream));
  GK_TRY(f64_deliver(h, q, out, true, h->tev[3], h->tev[4]));
  if (stats) {
    stats->n_graphs = N;
    stats->gram_path = 16;
    stats->gemm_launches = h->launches - launches0;
    stats->ms_gemm = ev_ms(h->tev[2], h->tev[3]);
    stats->ms_d2h = ev_ms(h->tev[3], h->tev[4]);
    stats->ms_total = stats->ms_gemm + stats->ms_d2h;
  }
  return GK_OK;
}

extern "C" {

int gk_svmt_draw(uint32_t* mt_key, int32_t* mt_pos, int64_t n_graphs, const int32_t* sizes, int32_t lo,
                 int32_t n_levels, const int32_t* counts, uint8_t* idx, int64_t n_idx) {
  if (!mt_key || !mt_pos || n_graphs < 0 || (n_graphs > 0 && (!sizes || !counts)) || n_levels < 1 || lo < 1)
    return fail(GK_ERR_ARG, "gk_svmt_draw: bad arguments");
  if (*mt_pos < 0 || *mt_pos > 624) return fail(GK_ERR_ARG, "gk_svmt_draw: MT19937 position outside [0, 624]");
  int64_t need = 0;
  for (int64_t g = 0; g < n_graphs; ++g) {
    if (sizes[g] < 1 || sizes[g] > SVMT_NMAX) return fail(GK_ERR_UNSUPPORTED, "gk_svmt_draw: a graph outside 1 .. 128 vertices");
    for (int li = 0; li < n_levels; ++li) {
      const int32_t v = counts[g * n_levels + li];
      if (v < 0) return fail(GK_ERR_ARG, "gk_svmt_draw: negative sample count");
      if (lo + li <= sizes[g]) need += (int64_t)v * (lo + li);
    }
  }
  if (need != n_idx || (need > 0 && !idx)) return fail(GK_ERR_ARG, "gk_svmt_draw: index buffer does not match the schedule");
  SvmtMT mt{mt_key, *mt_pos};
  uint8_t perm[SVMT_NMAX];
  int64_t o = 0;
  for (int64_t g = 0; g < n_graphs; ++g) {
    const int n = sizes[g];
    for (int li = 0; li < n_levels; ++li) {
      const int level = lo + li;
      if (level > n) continue;  // the reference sums all n alphas without drawing
      for (int32_t s = 0; s < counts[g * n_levels + li]; ++s) {
        mt.permutation(perm, n);
        memcpy(idx + o, perm, level);
        o += level;
      }
    }
  }
  *mt_pos = mt.pos;
  return GK_OK;
}

int gk_svmt_solve(gk_handle* h, int64_t n_graphs, const int32_t* sizes, const uint32_t* adj, gk_stats* stats) {
  if (!h) return fail(GK_ERR_ARG, "null handle");
  if (n_graphs < 1 || n_graphs > INT_MAX || !sizes || !adj) return fail(GK_ERR_ARG, "gk_svmt_solve: no graphs");
  std::vector<int> vptr(n_graphs + 1, 0);
  int nmax = 0;
  for (int64_t g = 0; g < n_graphs; ++g) {
    if (sizes[g] < 1) return fail(GK_ERR_ARG, "gk_svmt_solve: a graph without vertices");
    if (sizes[g] > SVMT_NMAX)
      return fail(GK_ERR_UNSUPPORTED, "gk_svmt_solve: a graph of more than 128 vertices (the eigenvalue workspace is "
                                      "n^2 doubles of shared memory)");
    if ((int64_t)vptr[g] + sizes[g] > INT_MAX) return fail(GK_ERR_UNSUPPORTED, "gk_svmt_solve: 2^31 or more vertices");
    vptr[g + 1] = vptr[g] + sizes[g];
    nmax = std::max(nmax, (int)sizes[g]);
  }
  const int64_t N = n_graphs, V = vptr[N];
  GK_CUDA(cudaSetDevice(h->dev));
  features_begin(h);
  h->svmt_sizes.clear();  // no solve until this call completes
  GK_TRY(h->svmt_vptr.ensure((size_t)(N + 1) * 4));
  GK_TRY(h->svmt_adj.ensure((size_t)V * 16));
  GK_TRY(h->svmt_m.ensure((size_t)N * 8));
  GK_TRY(h->svmt_alpha.ensure((size_t)V * 8));
  GK_TRY(h->svmt_iters.ensure((size_t)N * 4));
  GK_TRY(h->svmt_ctl.ensure(16));
  GK_CUDA(cudaEventRecord(h->tev[5], h->stream));
  GK_CUDA(cudaMemcpyAsync(h->svmt_vptr.p, vptr.data(), (size_t)(N + 1) * 4, cudaMemcpyHostToDevice, h->stream));
  GK_CUDA(cudaMemcpyAsync(h->svmt_adj.p, adj, (size_t)V * 16, cudaMemcpyHostToDevice, h->stream));
  GK_CUDA(cudaMemsetAsync(h->svmt_ctl.p, 0, 16, h->stream));
  GK_CUDA(cudaEventRecord(h->tev[0], h->stream));
  const size_t smem = ((size_t)nmax * nmax + 4 * (size_t)nmax) * 8;
  GK_CUDA(cudaFuncSetAttribute(svmt_eig, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int per_sm = 0;
  GK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, svmt_eig, SVMT_EIG_THREADS, smem));
  int grid = (int)std::min<int64_t>(N, (int64_t)h->sm_count * std::max(per_sm, 1));
  svmt_eig<<<grid, SVMT_EIG_THREADS, smem, h->stream>>>(h->svmt_vptr.as<int>(), h->svmt_adj.as<unsigned>(), (int)N,
                                                        h->svmt_m.as<double>());
  LAUNCH_CHECK(h);
  GK_CUDA(cudaEventRecord(h->tev[1], h->stream));
  GK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, svmt_smo, 32 * SVMT_SMO_WARPS, 0));
  grid = (int)std::min<int64_t>(cdiv(N, SVMT_SMO_WARPS), (int64_t)h->sm_count * std::max(per_sm, 1));
  svmt_smo<<<grid, 32 * SVMT_SMO_WARPS, 0, h->stream>>>(h->svmt_vptr.as<int>(), h->svmt_adj.as<unsigned>(), (int)N,
                                                        h->svmt_m.as<double>(), h->svmt_alpha.as<double>(),
                                                        h->svmt_iters.as<int>(), h->svmt_ctl.as<unsigned>());
  LAUNCH_CHECK(h);
  GK_CUDA(cudaEventRecord(h->tev[2], h->stream));
  h->svmt_sizes.assign(sizes, sizes + N);
  h->n_rows = 0;  // a new block starts without a row map
  if (stats) {
    memset(stats, 0, sizeof(*stats));
    stats->n_graphs = N; stats->n_vertices = V;
  }
  return GK_OK;
}

int gk_svmt_phi(gk_handle* h, int32_t lo, int32_t n_levels, const int32_t* counts, const uint8_t* idx, int64_t n_idx,
                const double* fit_phi0, int64_t n_fit, double* phi, double* m_out, double* alpha_out, int32_t* iters_out,
                gk_stats* stats) {
  if (!h) return fail(GK_ERR_ARG, "null handle");
  const int64_t N = (int64_t)h->svmt_sizes.size();
  if (N == 0) return fail(GK_ERR_STATE, "gk_svmt_phi: call gk_svmt_solve first");
  if (lo < 1 || n_levels < 1 || !counts || n_fit < 0 || (n_fit > 0 && !fit_phi0))
    return fail(GK_ERR_ARG, "gk_svmt_phi: bad arguments");
  std::vector<long long> off(2 * N);
  long long draws = 0, samples = 0;
  for (int64_t g = 0; g < N; ++g) {
    off[g] = draws; off[N + g] = samples;
    for (int li = 0; li < n_levels; ++li) {
      const int32_t v = counts[g * n_levels + li];
      if (v < 0) return fail(GK_ERR_ARG, "gk_svmt_phi: negative sample count");
      samples += v;
      if (lo + li <= h->svmt_sizes[g]) draws += (long long)v * (lo + li);
    }
  }
  if (draws != n_idx || (draws > 0 && !idx)) return fail(GK_ERR_ARG, "gk_svmt_phi: index buffer does not match the schedule");
  GK_CUDA(cudaSetDevice(h->dev));
  GK_TRY(h->svmt_cnt.ensure((size_t)N * n_levels * 4));
  GK_TRY(h->svmt_off.ensure((size_t)N * 16));
  GK_TRY(h->svmt_idx.ensure((size_t)std::max<long long>(draws, 1)));
  GK_TRY(h->svmt_sums.ensure((size_t)std::max<long long>(samples, 1) * 8));
  GK_TRY(h->svmt_phi.ensure((size_t)N * n_levels * 8));
  GK_TRY(h->svmt_rec.ensure((size_t)(n_fit + N) * 8));
  double* rec = h->svmt_rec.as<double>();
  GK_CUDA(cudaEventRecord(h->tev[7], h->stream));
  // word 0: the solve's SMO bit, word 1: this call's index bit
  GK_CUDA(cudaMemsetAsync(h->svmt_ctl.as<unsigned>() + 1, 0, 4, h->stream));
  GK_CUDA(cudaMemcpyAsync(h->svmt_cnt.p, counts, (size_t)N * n_levels * 4, cudaMemcpyHostToDevice, h->stream));
  GK_CUDA(cudaMemcpyAsync(h->svmt_off.p, off.data(), (size_t)N * 16, cudaMemcpyHostToDevice, h->stream));
  if (draws > 0) GK_CUDA(cudaMemcpyAsync(h->svmt_idx.p, idx, (size_t)draws, cudaMemcpyHostToDevice, h->stream));
  if (n_fit > 0) GK_CUDA(cudaMemcpyAsync(rec, fit_phi0, (size_t)n_fit * 8, cudaMemcpyHostToDevice, h->stream));
  GK_CUDA(cudaEventRecord(h->tev[3], h->stream));
  const long long* d_off = h->svmt_off.as<long long>();
  const int grid = (int)std::min<int64_t>(cdiv(N, SVMT_PHI_WARPS), (int64_t)h->sm_count * 16);
  svmt_phi<<<grid, 32 * SVMT_PHI_WARPS, 0, h->stream>>>(h->svmt_vptr.as<int>(), (int)N, h->svmt_alpha.as<double>(), lo,
                                                        n_levels, h->svmt_cnt.as<int>(), d_off, h->svmt_idx.as<unsigned char>(),
                                                        d_off + N, h->svmt_sums.as<double>(), h->svmt_phi.as<double>(),
                                                        rec + n_fit, h->svmt_ctl.as<unsigned>() + 1);
  LAUNCH_CHECK(h);
  GK_CUDA(cudaEventRecord(h->tev[4], h->stream));
  unsigned ctl[2] = {0, 0};
  GK_CUDA(cudaMemcpyAsync(ctl, h->svmt_ctl.p, 8, cudaMemcpyDeviceToHost, h->stream));
  if (phi) GK_CUDA(cudaMemcpyAsync(phi, h->svmt_phi.p, (size_t)N * n_levels * 8, cudaMemcpyDeviceToHost, h->stream));
  if (m_out) GK_CUDA(cudaMemcpyAsync(m_out, h->svmt_m.p, (size_t)N * 8, cudaMemcpyDeviceToHost, h->stream));
  int64_t nv = 0;
  for (int s : h->svmt_sizes) nv += s;
  if (alpha_out) GK_CUDA(cudaMemcpyAsync(alpha_out, h->svmt_alpha.p, (size_t)nv * 8, cudaMemcpyDeviceToHost, h->stream));
  if (iters_out) GK_CUDA(cudaMemcpyAsync(iters_out, h->svmt_iters.p, (size_t)N * 4, cudaMemcpyDeviceToHost, h->stream));
  GK_CUDA(cudaEventRecord(h->tev[6], h->stream));
  GK_CUDA(cudaStreamSynchronize(h->stream));
  const unsigned err = ctl[0] | ctl[1];
  if (err & SVMT_ERR_INDEX) return fail(GK_ERR_ARG, "gk_svmt_phi: a drawn index is not a vertex of its graph");
  if (err & SVMT_ERR_ITER)
    return fail(GK_ERR_RANGE, "SvmTheta: the one-class SMO did not converge within 10 000 000 iterations on a graph (libsvm "
                              "need not converge on a non-symmetric matrix)");
  h->svmt_nrec = n_fit + N;
  features_publish(h, FK_SVMT);
  if (stats) {
    stats->n_graphs = N; stats->n_vertices = nv;
    stats->ms_h2d = ev_ms(h->tev[5], h->tev[0]) + ev_ms(h->tev[7], h->tev[3]);
    stats->ms_features = ev_ms(h->tev[0], h->tev[1]);  // smallest eigenvalues
    stats->ms_rw = ev_ms(h->tev[1], h->tev[2]);        // SMO
    stats->ms_combine = ev_ms(h->tev[3], h->tev[4]);   // subset sums and phi
    stats->ms_d2h = ev_ms(h->tev[4], h->tev[6]);
  }
  return GK_OK;
}

}  // extern "C"

// ---------------------------------------------------------------------------
// GraphletSampling (graphlet_sampling.cuh), sampled route.  gk_gs_draw is host code on the estimator's MT19937 stream;
// gk_gs_features classifies the drawn samples on the device into the (graph, class) table, after the counts of the
// graphs before g0 handed back from an earlier run (a transform keeps the fit's samples without redrawing them).
// Table block gs_blk: keys [cap] u64 | counts [cap] u32 | sample counts [cap] u32 | class codes [cap] u32.
struct GsTable {
  unsigned long long* keys;
  unsigned *cnt, *raw, *code;
};

static GsTable gs_table(gk_handle* h) {
  GsTable t;
  char* b = h->gs_blk.as<char>();
  const size_t cap = h->gs_cap;
  t.keys = reinterpret_cast<unsigned long long*>(b);
  t.cnt = reinterpret_cast<unsigned*>(b + cap * 8);
  t.raw = t.cnt + cap;
  t.code = t.raw + cap;
  return t;
}

// gs_ctl: [error bits u32 | pad u32 | columns u64 | largest count u32 | entries u32]

// Gram of GraphletSampling (gram_path 17): the exact integer Gram of the (graph, column) table (gram_int: tensor
// cores, CUDA cores or no shared column), GK_NORMALIZE by the self similarities, which include the classes only the
// new graphs have (the reference's diagonal() over phi_y with its Y-only bins).
static int gram_gs(gk_handle* h, const GramReq& q, gk_stats* stats) {
  const GsTable t = gs_table(h);
  IntBlock fb;
  fb.keys = t.keys; fb.cnt = t.cnt; fb.cap = h->gs_cap;
  fb.colcnt = h->gs_colcnt.as<unsigned>(); fb.col_cap = h->gs_cols + 1; fb.n_columns = h->gs_cols;
  fb.diag = h->gs_diag.as<unsigned long long>();
  fb.part_max = h->gs_ctl.as<unsigned>() + 4; fb.part_new = fb.part_max + 1; fb.n_part = 1;
  fb.prologue_on_host = false;
  GK_TRY(gram_int(h, q, fb, stats));
  if (stats) stats->gram_path = 17;
  return GK_OK;
}

extern "C" {

int gk_gs_draw(uint32_t* mt_key, int32_t* mt_pos, int64_t n_graphs, const int32_t* sizes, int32_t k, int64_t n_samples,
               uint8_t* samp_size, int32_t* idx, int64_t idx_cap, int64_t* n_idx) {
  if (!mt_key || !mt_pos || n_graphs < 0 || (n_graphs > 0 && !sizes) || n_samples < 0 || !n_idx || k < 3)
    return fail(GK_ERR_ARG, "gk_gs_draw: bad arguments");
  if (*mt_pos < 0 || *mt_pos > 624) return fail(GK_ERR_ARG, "gk_gs_draw: MT19937 position outside [0, 624]");
  if (k > GS_KMAX) return fail(GK_ERR_UNSUPPORTED, "gk_gs_draw: graphlets of more than 6 vertices");
  int64_t need = 0;
  int nmax = 0;
  for (int64_t g = 0; g < n_graphs; ++g) {
    if (sizes[g] < 0) return fail(GK_ERR_ARG, "gk_gs_draw: a negative graph size");
    need += n_samples * std::min<int64_t>(k, sizes[g]);
    nmax = std::max(nmax, (int)sizes[g]);
  }
  if (need > idx_cap || (n_graphs * n_samples > 0 && !samp_size) || (need > 0 && !idx))
    return fail(GK_ERR_ARG, "gk_gs_draw: output buffers too small");
  SvmtMT mt{mt_key, *mt_pos};
  std::vector<int32_t> perm(std::max(nmax, 1));
  int64_t o = 0, s = 0;
  for (int64_t g = 0; g < n_graphs; ++g) {
    const int n = sizes[g], lo = std::min(3, n), hi = std::min<int>(k, n);
    for (int64_t t = 0; t < n_samples; ++t, ++s) {
      // rs.randint(min_r, max_r + 1) unless the range is one size, then rs.choice(n, r, replace=False)
      const int r = lo == hi ? lo : lo + (int)mt.interval((uint32_t)(hi - lo));
      mt.permutation(perm.data(), n);
      memcpy(idx + o, perm.data(), (size_t)r * 4);
      samp_size[s] = (uint8_t)r;
      o += r;
    }
  }
  *mt_pos = mt.pos;
  *n_idx = o;
  return GK_OK;
}

int gk_gs_features(gk_handle* h, int32_t k, int64_t n_fit, int64_t g0, const int64_t* samp_off,
                   const uint8_t* samp_size, const int32_t* idx, int64_t n_idx, const int64_t* prior, int64_t n_prior,
                   gk_stats* stats) {
  GK_TRY(need_packed(h, "gk_gs_features"));
  if (k < 1) return fail(GK_ERR_ARG, "gk_gs_features: k must be positive");
  if (k > GS_KMAX) return fail(GK_ERR_UNSUPPORTED, "gk_gs_features: graphlets of more than 6 vertices");
  const int64_t N = h->N;
  if (n_fit < 1 || n_fit > N || g0 < 0 || g0 > N || !samp_off || n_prior < 0 || (n_prior && !prior))
    return fail(GK_ERR_ARG, "gk_gs_features: bad arguments");
  const int64_t n_new = N - g0, S = samp_off[n_new];
  if (samp_off[0] != 0 || S < 0 || (S && !samp_size)) return fail(GK_ERR_ARG, "gk_gs_features: bad sample offsets");
  // every check on the host arguments before the first launch (the drawn indexes are checked on the device)
  const std::vector<int>& gp = h->graph_ptr_host;
  std::vector<long long> ioff(n_new + 1, 0);
  std::vector<long long> per_graph(n_new, 0);
  for (int64_t w = 0; w < n_new; ++w) {
    if (samp_off[w + 1] < samp_off[w]) return fail(GK_ERR_ARG, "gk_gs_features: bad sample offsets");
    if (samp_off[w + 1] - samp_off[w] >= (1LL << 31) - 1)
      return fail(GK_ERR_RANGE, "gk_gs_features: 2^31 or more samples of one graph (counts are u32)");
    long long t = 0;
    const int n = gp[g0 + w + 1] - gp[g0 + w];
    for (int64_t s = samp_off[w]; s < samp_off[w + 1]; ++s) {
      if (samp_size[s] > k || samp_size[s] > n) return fail(GK_ERR_ARG, "gk_gs_features: a sample larger than k or its graph");
      t += samp_size[s];
    }
    ioff[w + 1] = ioff[w] + t;
    per_graph[w] = samp_off[w + 1] - samp_off[w];
  }
  if (ioff[n_new] != n_idx || (n_idx && !idx)) return fail(GK_ERR_ARG, "gk_gs_features: index count does not match the sizes");
  for (int64_t i = 0; i < n_prior; ++i)
    if (prior[3 * i] < 0 || prior[3 * i] >= g0 || prior[3 * i + 1] < 0 || prior[3 * i + 1] >= gs_base(k + 1) ||
        prior[3 * i + 2] < 1 || prior[3 * i + 2] >= (1LL << 31) - 1)
      return fail(GK_ERR_ARG, "gk_gs_features: a bad prior count");
  const int64_t launches0 = h->launches;
  features_begin(h);
  GK_TRY(init_scalars(h, 0));
  GK_CUDA(cudaEventRecord(h->tev[2], h->stream));
  // ---- class table of the code space (sizes 0 .. k), and the number of classes it has
  const long long n_codes = gs_base(k + 1);
  static std::mutex classes_mu;
  static long long n_classes_of[GS_KMAX + 2] = {0};
  if (h->gs_canon_k < k) {
    GK_TRY(h->gs_canon.ensure((size_t)n_codes * 4));
    gs_canon<<<cdiv(n_codes, 256), 256, 0, h->stream>>>(n_codes, h->gs_canon.as<unsigned>());
    LAUNCH_CHECK(h);
    h->gs_canon_k = k;
    std::lock_guard<std::mutex> lk(classes_mu);
    if (!n_classes_of[k]) {
      std::vector<unsigned> c(n_codes);
      GK_CUDA(cudaMemcpyAsync(c.data(), h->gs_canon.p, (size_t)n_codes * 4, cudaMemcpyDeviceToHost, h->stream));
      GK_CUDA(cudaStreamSynchronize(h->stream));
      long long m = 0;
      for (long long x = 0; x < n_codes; ++x) m += c[x] == (unsigned)x;
      n_classes_of[k] = m;
    }
  }
  long long n_classes;
  {
    std::lock_guard<std::mutex> lk(classes_mu);
    n_classes = n_classes_of[k] ? n_classes_of[k] : n_codes;
  }
  GK_CUDA(cudaEventRecord(h->tev[3], h->stream));
  // ---- (graph, class) table: at most one entry per prior count and per sample or class of a graph
  long long bound = n_prior;
  for (int64_t w = 0; w < n_new; ++w) bound += std::min<long long>(per_graph[w], n_classes);
  const size_t cap = std::max<size_t>(next_pow2((size_t)std::max<long long>(bound, 1) * 2), 1024);
  if (cap > (1ULL << 31)) return fail(GK_ERR_RANGE, "gk_gs_features: (graph, class) table of 2^31 or more slots");
  h->gs_cap = cap;
  GK_TRY(h->gs_blk.ensure(cap * 20));
  GK_TRY(h->gs_first.ensure((size_t)n_codes * 8));
  GK_TRY(h->gs_colid.ensure((size_t)n_codes * 4));
  GK_TRY(h->gs_ctl.ensure(32));
  GK_TRY(h->gs_diag.ensure((size_t)N * 8));
  const size_t o_ioff = (size_t)(n_new + 1) * 8, o_size = o_ioff * 2, o_idx = (o_size + (size_t)S + 3) / 4 * 4;
  GK_TRY(h->gs_samp.ensure(o_idx + (size_t)n_idx * 4 + (size_t)std::max<int64_t>(n_prior, 1) * 24 + 16));
  const GsTable t = gs_table(h);
  unsigned* first_fit = h->gs_first.as<unsigned>();
  unsigned* first_new = first_fit + n_codes;
  unsigned* ctl = h->gs_ctl.as<unsigned>();
  char* sb = h->gs_samp.as<char>();
  const size_t o_prior = (o_idx + (size_t)n_idx * 4 + 7) / 8 * 8;
  GK_CUDA(cudaMemsetAsync(t.keys, 0xFF, cap * 8, h->stream));
  GK_CUDA(cudaMemsetAsync(t.cnt, 0, cap * 4, h->stream));
  GK_CUDA(cudaMemsetAsync(first_fit, 0xFF, (size_t)n_codes * 8, h->stream));
  GK_CUDA(cudaMemsetAsync(ctl, 0, 32, h->stream));
  GK_CUDA(cudaMemsetAsync(h->gs_diag.p, 0, (size_t)N * 8, h->stream));
  GK_CUDA(cudaMemcpyAsync(sb, samp_off, o_ioff, cudaMemcpyHostToDevice, h->stream));
  GK_CUDA(cudaMemcpyAsync(sb + o_ioff, ioff.data(), o_ioff, cudaMemcpyHostToDevice, h->stream));
  if (S) GK_CUDA(cudaMemcpyAsync(sb + o_size, samp_size, (size_t)S, cudaMemcpyHostToDevice, h->stream));
  if (n_idx) GK_CUDA(cudaMemcpyAsync(sb + o_idx, idx, (size_t)n_idx * 4, cudaMemcpyHostToDevice, h->stream));
  if (n_prior) {
    GK_CUDA(cudaMemcpyAsync(sb + o_prior, prior, (size_t)n_prior * 24, cudaMemcpyHostToDevice, h->stream));
    gs_prior<<<cdiv(n_prior, 256), 256, 0, h->stream>>>(n_prior, reinterpret_cast<const long long*>(sb + o_prior),
                                                        (int)n_fit, t.keys, t.cnt, (unsigned)(cap - 1), first_fit,
                                                        first_new);
    LAUNCH_CHECK(h);
  }
  GK_CUDA(cudaEventRecord(h->tev[0], h->stream));
  if (n_new > 0 && S > 0) {
    GsSampleParams p;
    p.g0 = (int)g0; p.g1 = (int)N;
    p.samp_off = reinterpret_cast<const long long*>(sb);
    p.idx_off = reinterpret_cast<const long long*>(sb + o_ioff);
    p.size = reinterpret_cast<const unsigned char*>(sb + o_size);
    p.idx = reinterpret_cast<const int*>(sb + o_idx);
    p.graph_ptr = h->graph_ptr.as<int>(); p.row_ptr = h->row_ptr.as<int>(); p.col_idx = h->col_idx.as<int>();
    p.canon = h->gs_canon.as<unsigned>();
    p.n_fit = (int)n_fit;
    p.keys = t.keys; p.cnt = t.cnt; p.mask = (unsigned)(cap - 1);
    p.first_fit = first_fit; p.first_new = first_new;
    p.err = ctl;
    const int grid = (int)std::min<int64_t>(cdiv(n_new, 8), (int64_t)h->sm_count * 16);
    gs_classify<<<grid, 256, 0, h->stream>>>(p);
    LAUNCH_CHECK(h);
  }
  GK_CUDA(cudaEventRecord(h->tev[1], h->stream));
  unsigned long long* n_cols = reinterpret_cast<unsigned long long*>(ctl + 2);
  gs_number<<<cdiv(n_codes, 256), 256, 0, h->stream>>>(n_codes, first_fit, first_new, h->gs_colid.as<unsigned>(), n_cols);
  LAUNCH_CHECK(h);
  unsigned hc[4] = {0, 0, 0, 0};
  GK_CUDA(cudaMemcpyAsync(hc, ctl, 16, cudaMemcpyDeviceToHost, h->stream));
  GK_CUDA(cudaStreamSynchronize(h->stream));
  if (hc[0] & 1u) return fail(GK_ERR_ARG, "gk_gs_features: a sample larger than 6 vertices");
  if (hc[0] & 2u) return fail(GK_ERR_ARG, "gk_gs_features: a drawn index is not a vertex of its graph");
  const int64_t M = (int64_t)(((unsigned long long)hc[3] << 32) | hc[2]);
  GK_TRY(h->gs_colcnt.ensure((size_t)(M + 1) * 4));
  GK_CUDA(cudaMemsetAsync(h->gs_colcnt.p, 0, (size_t)(M + 1) * 4, h->stream));
  const int sgrid = (int)std::min<int64_t>(cdiv((int64_t)cap, 256), (int64_t)h->sm_count * 16);
  gs_finish<<<sgrid, 256, 0, h->stream>>>(cap, (int)n_fit, first_fit, first_new, h->gs_colid.as<unsigned>(), t.keys,
                                          t.cnt, t.raw, t.code);
  LAUNCH_CHECK(h);
  nspd_level_stats<<<sgrid, 256, 0, h->stream>>>(cap, t.keys, t.cnt, h->gs_colcnt.as<unsigned>(),
                                                 h->gs_diag.as<unsigned long long>(), ctl + 4);
  LAUNCH_CHECK(h);
  GK_CUDA(cudaEventRecord(h->tev[4], h->stream));
  std::vector<unsigned long long> d(N);
  GK_CUDA(cudaMemcpyAsync(d.data(), h->gs_diag.p, (size_t)N * 8, cudaMemcpyDeviceToHost, h->stream));
  GK_CUDA(cudaMemcpyAsync(hc, ctl, 16, cudaMemcpyDeviceToHost, h->stream));
  GK_CUDA(cudaStreamSynchronize(h->stream));
  // K[i][j] <= sqrt(d_i d_j) <= max d: below 2^53 every entry and partial sum of the fp64 result is exact
  for (int64_t g = 0; g < N; ++g)
    if (d[g] >= (1ULL << 53))
      return fail(GK_ERR_RANGE, "GraphletSampling: a self similarity of 2^53 or more (K would not be exact in fp64)");
  h->gs_cols = M;
  h->n_columns = M;
  features_publish(h, FK_GS);
  if (stats) {
    memset(stats, 0, sizeof(*stats));
    stats->n_graphs = N; stats->n_vertices = h->V; stats->n_edges = h->E;
    stats->n_columns = M;
    stats->n_entries = S;
    stats->kernel_launches = h->launches - launches0;
    stats->ms_hash = ev_ms(h->tev[2], h->tev[3]);      // class table
    stats->ms_h2d = ev_ms(h->tev[3], h->tev[0]);       // samples to the device
    stats->ms_features = ev_ms(h->tev[0], h->tev[1]);  // classification and counts
    stats->ms_columns = ev_ms(h->tev[1], h->tev[4]);   // columns, "+1" rule, self similarities
  }
  return GK_OK;
}

int gk_gs_counts(gk_handle* h, int64_t cap, int64_t* out, int64_t* n_out) {
  if (!h || !n_out || (cap > 0 && !out)) return fail(GK_ERR_ARG, "gk_gs_counts: null argument");
  if (h->feature_kind != FK_GS) return fail(GK_ERR_STATE, "gk_gs_counts: run gk_gs_features first");
  GK_CUDA(cudaSetDevice(h->dev));
  const size_t tc = h->gs_cap;
  std::vector<char> b(tc * 20);
  GK_CUDA(cudaMemcpyAsync(b.data(), h->gs_blk.p, tc * 20, cudaMemcpyDeviceToHost, h->stream));
  GK_CUDA(cudaStreamSynchronize(h->stream));
  const unsigned long long* keys = reinterpret_cast<const unsigned long long*>(b.data());
  const unsigned* cnt = reinterpret_cast<const unsigned*>(b.data() + tc * 8);
  const unsigned *raw = cnt + tc, *code = raw + tc;
  std::vector<std::array<int64_t, 4>> rows;
  for (size_t i = 0; i < tc; ++i)
    if (keys[i] != EMPTY64) rows.push_back({(int64_t)(keys[i] >> 32), (int64_t)code[i], (int64_t)raw[i], (int64_t)cnt[i]});
  std::sort(rows.begin(), rows.end());
  *n_out = (int64_t)rows.size();
  if (cap >= (int64_t)rows.size())
    for (size_t i = 0; i < rows.size(); ++i) memcpy(out + 4 * i, rows[i].data(), 32);
  return GK_OK;
}

}  // extern "C"

extern "C" {

int gk_gram(gk_handle* h, int64_t n_fit, int32_t flags, int64_t row_begin, int64_t row_end, void* K_out,
            int32_t out_dtype, int64_t ld, double* xdiag, double* ydiag, gk_stats* stats) {
  if (!h) return fail(GK_ERR_ARG, "null handle");
  if (h->feature_kind == FK_NONE) return fail(GK_ERR_STATE, "gk_gram: no feature block (call gk_wl_features / gk_sp_features)");
  GramReq q;
  GK_TRY(gram_request(h, h->feature_kind, n_fit, flags, row_begin, row_end, K_out, out_dtype, ld, xdiag, ydiag, &q));
  GK_CUDA(cudaSetDevice(h->dev));
  return gram_route(h, q, stats);
}

int gk_set_row_map(gk_handle* h, int64_t n_rows, const int32_t* row_of_graph) {
  GK_TRY(need_packed(h, "gk_set_row_map"));
  if (n_rows <= 0 || !row_of_graph) {  // back to the identity
    h->n_rows = 0;
    return GK_OK;
  }
  for (int64_t g = 0; g < h->N; ++g)
    if (row_of_graph[g] < 0 || row_of_graph[g] >= n_rows) return fail(GK_ERR_ARG, "gk_set_row_map: row index out of range");
  GK_TRY(h->row_map.ensure(h->N * 4));
  GK_CUDA(cudaMemcpyAsync(h->row_map.p, row_of_graph, h->N * 4, cudaMemcpyHostToDevice, h->stream));
  GK_CUDA(cudaStreamSynchronize(h->stream));
  h->n_rows = n_rows;
  return GK_OK;
}

int gk_result_device(gk_handle* h, void** ptr, int64_t* rows, int64_t* cols, int64_t* ld, int32_t* dtype) {
  if (!h || !ptr) return fail(GK_ERR_ARG, "gk_result_device: null argument");
  if (!h->K.p || h->K_rows <= 0) return fail(GK_ERR_STATE, "gk_result_device: no device-resident result");
  *ptr = h->K.p;
  if (rows) *rows = h->K_rows;
  if (cols) *cols = h->K_cols;
  if (ld) *ld = h->K_ld;
  if (dtype) *dtype = h->K_dtype;
  return GK_OK;
}

int gk_fetch(gk_handle* h, void* K_out, int32_t out_dtype, int64_t ld) {
  if (!h || !K_out) return fail(GK_ERR_ARG, "gk_fetch: null argument");
  if (!h->K.p || h->K_rows <= 0) return fail(GK_ERR_STATE, "gk_fetch: no device-resident result");
  if (out_dtype != h->K_dtype) return fail(GK_ERR_ARG, "gk_fetch: dtype differs from the one gk_gram produced");
  const size_t esz = out_dtype == GK_F64 ? 8 : 4;
  if (ld <= 0) ld = h->K_cols;
  GK_CUDA(cudaSetDevice(h->dev));
  GK_CUDA(cudaMemcpy2DAsync(K_out, (size_t)ld * esz, h->K.p, (size_t)h->K_ld * esz, (size_t)h->K_cols * esz,
                            (size_t)h->K_rows, cudaMemcpyDeviceToHost, h->stream));
  GK_CUDA(cudaStreamSynchronize(h->stream));
  return GK_OK;
}

// --------------------------------------------------------------------------- TU files -> CSR (host only)
int gk_tu_open(const char* dir, const char* name, int32_t flags, gk_tu** out) {
  if (!dir || !name || !out) return fail(GK_ERR_ARG, "gk_tu_open: null argument");
  std::string err;
  const int r = gk::tu::open(dir, name, flags, out, &err);
  return r == GK_OK ? GK_OK : fail(r, "gk_tu_open: " + err);
}

int gk_tu_info(const gk_tu* t, int64_t* info) {
  if (!t || !info) return fail(GK_ERR_ARG, "gk_tu_info: null argument");
  info[0] = t->n_graphs; info[1] = t->n_nodes; info[2] = (int64_t)t->eu.size();
  info[3] = !t->node_label.empty(); info[4] = !t->el.empty(); info[5] = !t->classes.empty();
  info[6] = t->attr_dim; info[7] = 0;
  return GK_OK;
}

int gk_tu_pack(gk_tu* t, int32_t mode, int64_t* n_vertices, int64_t* n_edges) {
  if (!t) return fail(GK_ERR_ARG, "gk_tu_pack: null handle");
  std::string err;
  const int r = gk::tu::pack(t, mode, &err);
  if (r != GK_OK) return fail(r, "gk_tu_pack: " + err);
  if (n_vertices) *n_vertices = (int64_t)t->vnode.size();
  if (n_edges) *n_edges = (int64_t)t->col_idx.size();
  return GK_OK;
}

int gk_tu_fill(const gk_tu* t, int32_t* graph_ptr, int32_t* row_ptr, int32_t* col_idx, int32_t* node_labels,
               int32_t* edge_labels, double* attrs, int32_t* classes, int32_t* node_of_vertex) {
  if (!t) return fail(GK_ERR_ARG, "gk_tu_fill: null handle");
  if (t->mode < 0) return fail(GK_ERR_STATE, "gk_tu_fill: call gk_tu_pack first");
  const size_t V = t->vnode.size();
  if (graph_ptr) memcpy(graph_ptr, t->graph_ptr.data(), t->graph_ptr.size() * 4);
  if (row_ptr) memcpy(row_ptr, t->row_ptr.data(), t->row_ptr.size() * 4);
  if (col_idx && !t->col_idx.empty()) memcpy(col_idx, t->col_idx.data(), t->col_idx.size() * 4);
  if (node_labels) {
    if (t->vlabel.empty() && V) return fail(GK_ERR_STATE, "gk_tu_fill: the dataset has no node labels");
    if (V) memcpy(node_labels, t->vlabel.data(), V * 4);
  }
  if (edge_labels) {
    if (t->el.empty()) return fail(GK_ERR_STATE, "gk_tu_fill: the dataset has no edge labels");
    if (!t->elabel.empty()) memcpy(edge_labels, t->elabel.data(), t->elabel.size() * 4);
  }
  if (attrs) {
    if (!t->attr_dim) return fail(GK_ERR_STATE, "gk_tu_fill: node attributes were not loaded (GK_TU_ATTR_NODES)");
    for (size_t v = 0; v < V; ++v)
      memcpy(attrs + v * t->attr_dim, t->node_attr.data() + (size_t)t->vnode[v] * t->attr_dim, (size_t)t->attr_dim * 8);
  }
  if (classes) {
    if (t->classes.empty()) return fail(GK_ERR_STATE, "gk_tu_fill: the dataset has no graph classes");
    memcpy(classes, t->classes.data(), t->classes.size() * 4);
  }
  if (node_of_vertex)
    for (size_t v = 0; v < V; ++v) node_of_vertex[v] = t->vnode[v] + 1;
  return GK_OK;
}

int gk_tu_close(gk_tu* t) {
  delete t;
  return GK_OK;
}

// ---------------------------------------------------------------------------
}  // extern "C"

// ---------------------------------------------------------------------------
// The asynchronous WL pass: feature kernels, column statistics, the head/tail decision (gram_choose, ON THE DEVICE),
// panel, GEMM and tail are enqueued back to back -- the host synchronises once, at the end.  The synchronous route
// (gk_wl_features + gk_gram) needs the column histogram on the host between the two halves; here the host only sizes
// things by CAPACITY (the panel's row pitch, the tail buffers: what earlier passes on this handle allocated) and the
// device reports through GramDyn::bad when a capacity, an exactness bound or the WL hash check fails, in which case
// the caller repeats the pass through the synchronous route (which also grows the buffers).  Square fit_transform
// case with an fp32 device result: library-owned, caller's device buffer, or float64 host delivery.
static int wl_gram_async(gk_handle* h, int32_t n_iter, int32_t flags, void* K_out, int32_t out_dtype, int64_t ld,
                         double* xdiag, gk_stats* stats, bool* done) {
  *done = false;
  for (const char* name : {"GRAKEL_B200_NO_ASYNC", "GRAKEL_B200_PROF", "GRAKEL_B200_WL_FUSED",
                           "GRAKEL_B200_CTA2", "GRAKEL_B200_NO_TMA_STORE", "GRAKEL_B200_WIDEN", "GRAKEL_B200_NO_TRI",
                           "GRAKEL_B200_MIRROR_TMA", "GRAKEL_B200_DEBUG"})
    if (getenv(name)) return GK_OK;
  if (flags & ~(GK_OUT_DEVICE | GK_DENSE_ALL)) return GK_OK;
  if (h->N <= 0 || !h->has_labels || h->V == 0 || n_iter < 0 || n_iter + 1 >= MAX_LEVELS || h->n_rows > 0) return GK_OK;
  const int64_t N = h->N, V = h->V;
  const bool dev_out = (flags & GK_OUT_DEVICE) != 0;
  const bool host_out = K_out && !dev_out;
  if (host_out && out_dtype != GK_F64) return GK_OK;
  if (!host_out && out_dtype != GK_F32) return GK_OK;
  if (dev_out && !K_out) return GK_OK;
  if (ld > 0 && ld < N) return GK_OK;  // (the synchronous route reports the error)
  if (dev_out && (((uintptr_t)K_out) % 16 != 0 || ((ld > 0 ? ld : N) * 4) % 16 != 0)) return GK_OK;
  // panel type: u8 unless the switch is off or the last Gram on this handle saw a count of 256 (the device checks the
  // counts of THIS pass against the type and sends it to the synchronous route if one does not fit)
  const int elem_bytes = (u8_panel_enabled() && h->last_max_count <= 255) ? 1 : 2;
  const int bk = panel_bk(elem_bytes);
  // capacities left by earlier passes, reasoned in bytes (passes of either panel type share the buffer): row pitch
  // S_bytes, a whole number of 128-byte k-blocks
  int64_t S_bytes = (int64_t)(h->panel.cap / (size_t)N) / 128 * 128;
  {  // no wider than the last cost-model pass needed, plus a quarter (a dense-all pass may have left a much larger buffer,
     // and the whole pitch is zeroed)
    const long long want = h->head_row_bytes;
    if (!(flags & GK_DENSE_ALL) && !getenv("GRAKEL_B200_FORCE_T") && want > 0)
      S_bytes = std::min<int64_t>(S_bytes, (want + want / 4 + 127) / 128 * 128 + 128);
  }
  const int64_t S = S_bytes / elem_bytes;  // row pitch in elements
  if (S_bytes < 128 || !h->tail_desc.p || !h->tail_cur.p || !h->tail_ent.p) return GK_OK;
  const long long cap_tail_cols = (long long)std::min(h->tail_desc.cap / sizeof(int2), h->tail_cur.cap / 4);
  const long long cap_tail_ent = (long long)(h->tail_ent.cap / sizeof(int2));
  GK_CUDA(cudaSetDevice(h->dev));
  const int L = n_iter + 1;
  features_begin(h);
  h->n_levels = L;
  const int64_t launches0 = h->launches;
  WlPlan pl;
  GK_TRY(wl_setup(h, n_iter, &pl));
  if (!pl.fused) return GK_OK;
  const int64_t D = (int64_t)h->n_labels0 + V * (int64_t)(L - 1);
  FeatStats fst;
  GK_TRY(reset_feature_stats(h, D + 1, (int64_t)std::max(pl.nb, pl.G) * L, &fst, false));
  GK_TRY(h->colstats.ensure(sizeof(ColStats)));
  if (!h->gram_dyn.p) {
    GK_TRY(h->gram_dyn.ensure(sizeof(GramDyn)));
    GK_CUDA(cudaMemsetAsync(h->gram_dyn.p, 0, sizeof(GramDyn), h->stream));  // the block ticket starts at zero
  }
  DevScalars* sc = h->scalars.as<DevScalars>();
  ColStats* cs = h->colstats.as<ColStats>();
  GramDyn* dyn = h->gram_dyn.as<GramDyn>();
  // ---- features first: everything else the host has to prepare overlaps the WL kernel
  GK_CUDA(cudaMemsetAsync(cs, 0, sizeof(ColStats), h->stream));
  GK_CUDA(cudaEventRecord(h->tev[2], h->stream));
  const unsigned long long seed = mix64(0x5851F42D4C957F2DULL);
  GK_TRY(wl_launch_v2(h, pl, seed, wl_take_degen(h), fst, false));
  h->wl_sparse_ids = L > 1;
  GK_CUDA(cudaEventRecord(h->tev[3], h->stream));
  // ---- the panel (full row pitch) is zeroed on the side stream while the column statistics run (the WL kernel itself
  // owns every register file: nothing can share an SM with it)
  GK_CUDA(cudaEventRecord(h->ev_fork, h->stream));
  GK_CUDA(cudaStreamWaitEvent(h->stream2, h->ev_fork, 0));
  panel_zero_rows<<<h->sm_count * 4, 256, 0, h->stream2>>>(h->panel.as<unsigned char>(), N, S_bytes, (int)(S_bytes / 16));
  LAUNCH_CHECK(h);
  GK_CUDA(cudaEventRecord(h->ev_stage[0], h->stream2));

  GK_TRY(h->colslot.ensure(std::max<int64_t>(D, 1) * 4));
  GK_TRY(h->h_dyn.ensure(sizeof(GramDyn) + 64));
  GK_TRY(h->diag_f64.ensure(N * 8));
  // output
  void* d_out;
  long long d_ld;
  if (dev_out) {
    d_out = K_out;
    d_ld = ld > 0 ? ld : N;
  } else {
    h->K_ld = (N + 7) / 8 * 8;
    GK_TRY(h->K.ensure((size_t)N * h->K_ld * 4));
    d_out = h->K.p;
    d_ld = h->K_ld;
    h->K_rows = N; h->K_cols = N; h->K_dtype = GK_F32;
  }
  // tile list (same key as gk_gram's)
  {
    const long long tkey[8] = {0, 0, (long long)N, 0, (long long)N, 1, BM2, 0};
    if (memcmp(tkey, h->tiles_key, sizeof(tkey)) != 0 || !h->tiles.p) {
      std::vector<int2> tiles;
      build_tiles(tiles, 0, (int)N, 0, (int)N, true, BM2);
      GK_TRY(h->h_tiles.ensure(tiles.size() * sizeof(int2) + 16));
      memcpy(h->h_tiles.p, tiles.data(), tiles.size() * sizeof(int2));
      GK_TRY(h->tiles.ensure(tiles.size() * sizeof(int2) + 16));
      GK_CUDA(cudaMemcpyAsync(h->tiles.p, h->h_tiles.p, tiles.size() * sizeof(int2), cudaMemcpyHostToDevice, h->stream));
      memcpy(h->tiles_key, tkey, sizeof(tkey));
      h->tiles_n = (long long)tiles.size();
    }
  }
  const int64_t n_tiles = h->tiles_n;
  CUtensorMap tmA, tmC;
  PeerMaps peer_maps;
  memset(&peer_maps, 0, sizeof(peer_maps));
  GK_TRY(make_panel_map(&tmA, h->panel.p, S, N, BM, elem_bytes));
  GK_TRY(make_out_map(&tmC, d_out, N, N, d_ld));
  int force_T = (flags & GK_DENSE_ALL) ? 1 : -1;
  if (force_T < 0) {
    const char* e = getenv("GRAKEL_B200_FORCE_T");
    if (e && *e) force_T = std::max(1, atoi(e));
  }
  // ---- columns: self similarities, histogram, the decision -- one launch, one copy back
  GK_CUDA(cudaEventRecord(h->tev[4], h->stream));
  const int64_t Dn = std::max<int64_t>(D, 1);
  const int nbc = cdiv(Dn, 256);
  {
    ColFusedParams q;
    q.D = Dn; q.N = (int)N; q.L = L;
    q.colcnt = h->colcnt.as<unsigned>();
    q.diag = h->diag_u64.as<unsigned long long>(); q.diag_f64 = h->diag_f64.as<double>();
    q.n_part = (int)h->n_part; q.part_max = h->part_max.as<unsigned>(); q.part_new = h->part_new.as<unsigned>();
    q.cs = cs; q.sc = sc; q.dyn = dyn;
    q.flops_per_col = (double)N * (double)(N + 1); q.rate = panel_rate(elem_bytes); q.t_atomic = COST_T_ATOMIC;
    q.force_T = force_T; q.stride_cap = (int)S; q.bk = bk;
    q.max_panel_count = elem_bytes == 1 ? 255u : 256u;
    q.cap_tail_cols = cap_tail_cols; q.cap_tail_ent = cap_tail_ent;
    col_stats_fused<<<h->sm_count * 4, 256, 0, h->stream>>>(q);
    LAUNCH_CHECK(h);
  }
  // the copy back travels on the side stream: the main stream goes straight on to the classification
  GK_CUDA(cudaEventRecord(h->ev_stage[1], h->stream));
  GK_CUDA(cudaStreamWaitEvent(h->stream2, h->ev_stage[1], 0));
  GK_CUDA(cudaMemcpyAsync(h->h_dyn.p, dyn, sizeof(GramDyn), cudaMemcpyDeviceToHost, h->stream2));
  GK_CUDA(cudaEventRecord(h->ev_join, h->stream2));  // the host waits for THIS, not for the GEMM behind it
  unsigned* col_counters = reinterpret_cast<unsigned*>(cs);  // cleared by the deciding block
  col_classify<<<nbc, 256, 0, h->stream>>>(Dn, 1, (int)N, h->colcnt.as<unsigned>(), nullptr, nullptr, 1, h->colslot.as<int>(),
                                           h->tail_desc.as<int2>(), h->tail_cur.as<unsigned>(), col_counters, dyn);
  LAUNCH_CHECK(h);
  GK_CUDA(cudaStreamWaitEvent(h->stream, h->ev_stage[0], 0));  // the zeroed panel
  if (elem_bytes == 1)
    feat_scatter<<<cdiv((long long)h->ft_cap, 256), 256, 0, h->stream>>>(
        h->ft_cap, h->ft_keys.as<unsigned long long>(), h->ft_cnt.as<unsigned>(), h->colslot.as<int>(), nullptr,
        h->panel.as<uint8_t>(), S, h->tail_cur.as<unsigned>(), h->tail_desc.as<int2>(), h->tail_ent.as<int2>());
  else
    feat_scatter<<<cdiv((long long)h->ft_cap, 256), 256, 0, h->stream>>>(
        h->ft_cap, h->ft_keys.as<unsigned long long>(), h->ft_cnt.as<unsigned>(), h->colslot.as<int>(), nullptr,
        h->panel.as<__nv_bfloat16>(), S, h->tail_cur.as<unsigned>(), h->tail_desc.as<int2>(), h->tail_ent.as<int2>());
  LAUNCH_CHECK(h);
  // ---- tail: bucketed by 32 x 32 block of K for the GEMM epilogue (GRAKEL_B200_TAIL_FUSED=0: the separate tail_pairs kernel)
  const char* e_tf = getenv("GRAKEL_B200_TAIL_FUSED");
  const bool tail_fused = !(e_tf && atoi(e_tf) == 0);
  const int nb32 = (int)((N + 31) / 32);
  const unsigned ovf_cap = 1u << 20;
  const char* e_sym = getenv("GRAKEL_B200_TB_SYM");
  const int tb_sym = (e_sym && atoi(e_sym) != 0) ? 1 : 0;  // symmetric lists (pairs with row < column only): half the atomics
  int tb_cap = TB_CAP;  // tests shrink it (GRAKEL_B200_TB_CAP) to drive updates through the overflow list
  if (const char* e = getenv("GRAKEL_B200_TB_CAP")) tb_cap = std::max(0, std::min(TB_CAP, atoi(e)));
  unsigned* d_ovf_n = nullptr;
  unsigned* d_tb_cnt_all = nullptr;
  if (tail_fused) {
    const size_t n_blk = (size_t)nb32 * nb32;
    // one buffer, one memset: [entry lines (n_blk x 128 B) | block counters | overflow counter]
    const size_t tb_words = n_blk * TB_CAP + n_blk + 16;
    GK_TRY(h->tb_ent.ensure(tb_words * 4));
    GK_TRY(h->tb_ovf.ensure((size_t)ovf_cap * sizeof(int4)));
    unsigned* d_tb_cnt = h->tb_ent.as<unsigned>() + n_blk * TB_CAP;
    d_tb_cnt_all = d_tb_cnt;
    d_ovf_n = d_tb_cnt + n_blk;
    GK_CUDA(cudaMemsetAsync(h->tb_ent.p, 0, tb_words * 4, h->stream));
    tail_bucket<<<h->sm_count * 16, 256, 0, h->stream>>>(h->tail_desc.as<int2>(), h->tail_ent.as<int2>(), dyn, nb32, tb_cap, TB_CAP, tb_sym,
                                                         d_tb_cnt, h->tb_ent.as<unsigned>(), h->tb_ovf.as<int4>(), ovf_cap, d_ovf_n);
    LAUNCH_CHECK(h);
    GK_CUDA(cudaMemcpyAsync(reinterpret_cast<char*>(h->h_dyn.p) + sizeof(GramDyn), d_ovf_n, 4, cudaMemcpyDeviceToHost, h->stream));
  }
  // ---- GEMM (k extent read from the device) + tail
  GramParams p;
  memset(&p, 0, sizeof(p));
  p.a_row_end = (int)N; p.b_row_end = (int)N;
  p.out = d_out; p.ld = d_ld;
  p.mirror = 2;
  p.fix_diag = 1;
  p.vec_ok = (((uintptr_t)d_out) % 32 == 0 && (d_ld * 4) % 32 == 0) ? 1 : 0;
  p.diag = h->diag_f64.as<double>();
  p.tma_store = 1;
  p.tiles = h->tiles.as<int2>();
  p.n_tiles = (int)n_tiles;
  p.num_k_blocks = 1;
  p.nkb_dev = &dyn->num_k_blocks;
  if (tail_fused) { p.tb_cnt = d_tb_cnt_all; p.tb_ent = h->tb_ent.as<unsigned>(); p.tb_nb32 = nb32; p.tb_cap = tb_cap; p.tb_sym = tb_sym; }
  const int grid = 2 * (int)std::min<int64_t>(n_tiles, h->sm_count / 2);
  GK_CUDA(cudaEventRecord(h->tev[6], h->stream));
  if (elem_bytes == 1) gram_tc2_kernel<2><<<grid, GEMM_THREADS, GEMM2_SMEM, h->stream>>>(tmA, tmC, p, peer_maps);
  else gram_tc2_kernel<0><<<grid, GEMM_THREADS, GEMM2_SMEM, h->stream>>>(tmA, tmC, p, peer_maps);
  LAUNCH_CHECK(h);
  GK_CUDA(cudaEventRecord(h->tev[7], h->stream));
  if (tail_fused)
    tail_overflow_apply<<<64, 256, 0, h->stream>>>(h->tb_ovf.as<int4>(), d_ovf_n, ovf_cap, (float*)d_out, d_ld, tb_sym);
  else
    tail_pairs<float><<<h->sm_count * 16, 256, 0, h->stream>>>(0, h->tail_desc.as<int2>(), h->tail_ent.as<int2>(), (int)N, 1, 0, (int)N,
                                                              (float*)d_out, d_ld, dyn);
  LAUNCH_CHECK(h);
  GK_CUDA(cudaEventRecord(h->ev[13], h->stream));
  const int64_t launches_all = h->launches - launches0;

  // ---- the decision reaches the host while the GEMM runs
  GK_CUDA(cudaEventSynchronize(h->ev_join));
  const GramDyn hd = *h->h_dyn.as<GramDyn>();
  if (hd.bad) {  // repeat through the synchronous route (it reports errors, retries hash seeds, grows buffers)
    GK_CUDA(cudaStreamSynchronize(h->stream));
    return GK_OK;
  }
  GK_CUDA(cudaEventRecord(h->ev[14], h->stream));
  if (host_out) GK_TRY(deliver_square(h, reinterpret_cast<const float*>(d_out), d_ld, N, reinterpret_cast<double*>(K_out), ld > 0 ? ld : N,
                                      (int64_t)hd.max_diag));
  if (xdiag) GK_CUDA(cudaMemcpyAsync(xdiag, h->diag_f64.p, N * 8, cudaMemcpyDeviceToHost, h->stream));
  GK_CUDA(cudaEventRecord(h->ev[15], h->stream));
  GK_CUDA(cudaStreamSynchronize(h->stream));
  if (tail_fused && *reinterpret_cast<const unsigned*>(reinterpret_cast<const char*>(h->h_dyn.p) + sizeof(GramDyn)) > ovf_cap)
    return GK_OK;  // more block overflows than the list holds (never seen): the synchronous route recomputes everything
  // ---- state as gk_wl_features + gk_gram leave it
  h->n_columns = hd.n_columns;
  h->Dc = hd.Dc; h->Dc_pad = hd.Dc_pad;
  if (force_T < 0) h->head_row_bytes = (long long)hd.Dc_pad * elem_bytes;
  h->last_max_count = (long long)hd.max_count;
  h->pro_hist = hd.hist;
  h->pro_max_count = (long long)hd.max_count; h->pro_max_diag = (long long)hd.max_diag; h->pro_n_entries = (long long)hd.n_entries;
  h->pro_ready = true;
  features_publish(h, FK_WL);
  if (stats) {
    memset(stats, 0, sizeof(*stats));
    stats->n_graphs = N; stats->n_vertices = V; stats->n_edges = h->E;
    stats->n_levels = L;
    for (int i = 0; i < L; ++i) { stats->level_dims[i] = hd.level_dims[i]; stats->n_columns += hd.level_dims[i]; }
    if (L == 1) stats->n_columns = h->n_columns;
    stats->hash_retries = 0;
    stats->kernel_launches = launches_all;
    stats->ms_features = ev_ms(h->tev[2], h->tev[3]);
    stats->n_entries = (int64_t)hd.n_entries;
    stats->n_dense_columns = hd.Dc;
    stats->n_tail_columns = hd.n_tail_cols;
    stats->tail_updates = (int64_t)hd.tail_work;
    stats->threshold = hd.T;
    stats->max_count = (int64_t)hd.max_count;
    stats->max_diag = (int64_t)hd.max_diag;
    stats->gram_path = 1;
    stats->gemm_elem_bytes = elem_bytes;
    stats->gemm_tiles = n_tiles;
    stats->gemm_launches = 0;
    stats->ms_panel = ev_ms(h->tev[4], h->tev[6]);
    stats->ms_gemm = ev_ms(h->tev[6], h->tev[7]);
    stats->ms_tail = ev_ms(h->tev[7], h->ev[13]);
    stats->ms_d2h = ev_ms(h->ev[14], h->ev[15]);
    stats->ms_total = ev_ms(h->tev[2], h->ev[15]);
  }
  *done = true;
  return GK_OK;
}

extern "C" {

// WL features + square Gram in one call on the packed block (gk_wl_features followed by gk_gram(n_fit = N)): the
// asynchronous pass above when it applies, else the two synchronous calls.
int gk_wl_gram(gk_handle* h, int32_t n_iter, int32_t flags, void* K_out, int32_t out_dtype, int64_t ld, double* xdiag,
               gk_stats* stats) {
  if (!h) return fail(GK_ERR_ARG, "null handle");
  if (out_dtype != GK_F32 && out_dtype != GK_F64) return fail(GK_ERR_ARG, "gk_wl_gram: bad out_dtype");
  bool done = false;
  GK_TRY(wl_gram_async(h, n_iter, flags, K_out, out_dtype, ld, xdiag, stats, &done));
  if (done) return GK_OK;
  gk_stats s1, s2;
  memset(&s1, 0, sizeof(s1));
  GK_TRY(gk_wl_features(h, n_iter, &s1));
  s2 = s1;
  GK_TRY(gk_gram(h, h->N, flags, 0, -1, K_out, out_dtype, ld, xdiag, nullptr, &s2));
  if (stats) {
    *stats = s2;
    stats->kernel_launches = s1.kernel_launches;
  }
  return GK_OK;
}

int gk_wl_fit_transform(gk_handle* h, int64_t n_graphs, const int32_t* graph_ptr, const int32_t* row_ptr,
                        const int32_t* col_idx, const int32_t* labels, int32_t n_iter, int32_t flags, void* K_out,
                        int32_t out_dtype, int64_t ld, double* diag, gk_stats* stats) {
  gk_stats st;
  memset(&st, 0, sizeof(st));
  GK_TRY(gk_pack_csr(h, n_graphs, graph_ptr, row_ptr, col_idx, labels, nullptr, nullptr, 0));
  GK_TRY(gk_wl_gram(h, n_iter, flags, K_out, out_dtype, ld, diag, &st));
  if (stats) {
    *stats = st;
    stats->ms_h2d = ev_ms(h->tev[0], h->tev[1]);
  }
  return GK_OK;
}

int gk_sp_fit_transform(gk_handle* h, int64_t n_graphs, const int32_t* graph_ptr, const int32_t* row_ptr,
                        const int32_t* col_idx, const int32_t* labels, const double* weights, int32_t sp_flags,
                        int32_t flags, void* K_out, int32_t out_dtype, int64_t ld, double* diag, gk_stats* stats) {
  gk_stats s1, s2;
  memset(&s1, 0, sizeof(s1));
  GK_TRY(gk_pack_csr(h, n_graphs, graph_ptr, row_ptr, col_idx, labels, weights, nullptr, 0));
  GK_TRY(gk_sp_features(h, sp_flags, &s1));
  s2 = s1;
  GK_TRY(gk_gram(h, n_graphs, flags, 0, -1, K_out, out_dtype, ld, diag, nullptr, &s2));
  if (stats) {
    *stats = s2;
    stats->kernel_launches = s1.kernel_launches;
    stats->ms_h2d = ev_ms(h->tev[0], h->tev[1]);
  }
  return GK_OK;
}

// ---------------------------------------------------------------------------
// Dense self-test of the two Gram kernels (tests only): counts[n x d] -> K = C C^T.
int gk_selftest_gram(gk_handle* h, int64_t n, int64_t d, const uint16_t* counts, double* out_tc, double* out_simt) {
  if (!h || !counts || n <= 0 || d <= 0) return fail(GK_ERR_ARG, "gk_selftest_gram: bad arguments");
  GK_CUDA(cudaSetDevice(h->dev));
  // the panel type gk_gram would choose: u8 when every count is <= 255 (and the switch is on), else bf16
  unsigned max_c = 0;
  for (int64_t i = 0; i < n * d; ++i) max_c = std::max<unsigned>(max_c, counts[i]);
  const int elem_bytes = (u8_panel_enabled() && max_c <= 255) ? 1 : 2;
  const int bk = panel_bk(elem_bytes);
  const int64_t dpad = (d + bk - 1) / bk * bk;
  std::vector<uint8_t> pb((size_t)n * dpad * elem_bytes, 0);
  std::vector<unsigned> pu((size_t)n * d, 0u);
  std::vector<double> dg(n, 0.0);
  for (int64_t i = 0; i < n; ++i)
    for (int64_t j = 0; j < d; ++j) {
      const unsigned c = counts[i * d + j];
      if (elem_bytes == 1) pb[i * dpad + j] = (uint8_t)c;
      else reinterpret_cast<__nv_bfloat16*>(pb.data())[i * dpad + j] = __float2bfloat16((float)c);
      pu[i * d + j] = c;
      dg[i] += (double)c * c;
    }
  gk::DevBuf dpb, dpu, ddg, dk1, dk2, dtl;
  GK_TRY(dpb.ensure(pb.size()));
  GK_TRY(dpu.ensure(pu.size() * 4));
  GK_TRY(ddg.ensure(n * 8));
  GK_TRY(dk1.ensure((size_t)n * n * 8));
  GK_TRY(dk2.ensure((size_t)n * n * 8));
  GK_CUDA(cudaMemcpyAsync(dpb.p, pb.data(), pb.size(), cudaMemcpyHostToDevice, h->stream));
  GK_CUDA(cudaMemcpyAsync(dpu.p, pu.data(), pu.size() * 4, cudaMemcpyHostToDevice, h->stream));
  GK_CUDA(cudaMemcpyAsync(ddg.p, dg.data(), n * 8, cudaMemcpyHostToDevice, h->stream));
  GK_CUDA(cudaMemsetAsync(dk1.p, 0xFF, (size_t)n * n * 8, h->stream));  // NaN pattern: unwritten entries show up
  GK_CUDA(cudaMemsetAsync(dk2.p, 0xFF, (size_t)n * n * 8, h->stream));
  GramParams p;
  memset(&p, 0, sizeof(p));
  p.a_row_end = (int)n; p.b_row_end = (int)n;
  p.ld = n;
  p.diag = ddg.as<double>();
  p.vec_ok = (n * 8) % 32 == 0;
  int rc = GK_OK;
  if (out_tc) {
    std::vector<int2> tiles;
    build_tiles(tiles, 0, (int)n, 0, (int)n, true, BM);
    GK_TRY(dtl.ensure(tiles.size() * sizeof(int2)));
    GK_CUDA(cudaMemcpyAsync(dtl.p, tiles.data(), tiles.size() * sizeof(int2), cudaMemcpyHostToDevice, h->stream));
    CUtensorMap tmA, tmB, tmC;
    memset(&tmC, 0, sizeof(tmC));
    GK_TRY(make_panel_map(&tmA, dpb.p, dpad, n, BM, elem_bytes));
    GK_TRY(make_panel_map(&tmB, dpb.p, dpad, n, BN, elem_bytes));
    p.tiles = dtl.as<int2>();
    p.n_tiles = (int)tiles.size();
    p.num_k_blocks = (int)(dpad / bk);
    p.out = dk1.p;
    p.mirror = 1;
    launch_tc<double, false>(h, tmA, tmB, tmC, p, (int)std::min<size_t>(tiles.size(), h->sm_count), elem_bytes);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
    if (e != cudaSuccess) rc = fail(GK_ERR_CUDA, std::string("selftest tensor-core kernel: ") + cudaGetErrorString(e));
    else {
      GK_CUDA(cudaMemcpy(out_tc, dk1.p, (size_t)n * n * 8, cudaMemcpyDeviceToHost));
    }
  }
  if (rc == GK_OK && out_simt) {
    p.out = dk2.p;
    p.mirror = 0;
    launch_simt<double, false>(h, dpu.as<unsigned>(), d, (int)d, 0, (int)n, 0, (int)n, p);
    GK_CUDA(cudaGetLastError());
    GK_CUDA(cudaStreamSynchronize(h->stream));
    GK_CUDA(cudaMemcpy(out_simt, dk2.p, (size_t)n * n * 8, cudaMemcpyDeviceToHost));
  }
  return rc;
}

int gk_selftest_live_bytes(int64_t* device, int64_t* pinned) {
  if (!device || !pinned) return fail(GK_ERR_ARG, "gk_selftest_live_bytes: null argument");
  *device = g_live_bytes[0];
  *pinned = g_live_bytes[1];
  return GK_OK;
}

}  // extern "C"
