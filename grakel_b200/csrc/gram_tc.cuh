// Gram matrix K = A * B^T over the dense integer feature panel on Hopper's tensor cores
// (wgmma.mma_async, accumulators in registers, operands staged by TMA with the
// 128-byte swizzle).  Replaces `self.X.dot(self.X.T)` / `Y[:, :D].dot(self.X.T)`
// (vertex_histogram.py:177-179), the per-level `np.sum` (weisfeiler_lehman.py:270)
// and `np.dot(phi_x, phi_x.T)` (shortest_path.py:404) of the reference.
//
// Operand types (KIND): the panel holds integer counts, as u8 when every count is <= 255
// (KIND 2: u8 x u8 -> s32, exact integer accumulation, twice the bf16 MMA rate) and as
// bf16 when a count is 256 (KIND 0: bf16 x bf16 -> f32; products and partial sums are
// integers < 2^24, exact in fp32).  Either way the host checks that every self similarity
// -- and hence every entry of K -- is below 2^24 before choosing this path, so the fp32
// result is exact and bit-identical to the reference's float64 arithmetic.  KIND 1 (tf32)
// serves the split-precision real-valued Gram of ShortestPathAttr.
//
// Kernel shape (one persistent CTA per SM, 384 threads = three warpgroups):
//   warpgroup 0     TMA producer (one elected thread); runs ahead into the next tile
//                   while the consumers drain their accumulators
//   warpgroups 1-2  wgmma m64n256 over 64 rows each of the 128 x 256 tile,
//                   then the epilogue of those rows (diagonal fix / normalise -> global,
//                   plus the mirrored tile for the symmetric case)
// smem: 4 stages x (A 128 + B 256 rows of one 128-byte k-block: 64 bf16 or 128 u8) = 192 KiB,
// mbarrier ring, 32 KiB of epilogue staging (two 32x32 fp32 tiles per pair of warps).
#pragma once
#include "common.cuh"

namespace gk {

constexpr int BM = 128, BN = 256, BK = 64;
constexpr int STAGES = 4;
constexpr int A_BYTES = BM * BK * 2;
constexpr int B_BYTES = BN * BK * 2;
constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
constexpr int BK_TF32 = 32;  // tf32 operands: 32 elements per 128-byte k-block
constexpr int BK_U8 = 128;   // u8 operands: 128 elements per 128-byte k-block
constexpr int GEMM_THREADS = 384;
// epilogue staging for TMA stores: per pair of consumer warps (one 32-row block) two 32x32 fp32 tiles
constexpr int EPI_BUF_BYTES = 32 * 32 * 4;
constexpr int EPI_BYTES = 4 * 2 * EPI_BUF_BYTES;
constexpr int GEMM_SMEM = STAGES * STAGE_BYTES + 1024 /*align*/ + 1024 /*barriers*/ + EPI_BYTES;
static_assert(GEMM_SMEM <= 232448, "shared memory budget of one CTA");

struct GramParams {
  const int2* tiles;   // {first A row, first B row} in panel-row (graph) coordinates
  int n_tiles;
  int num_k_blocks;    // Dc_pad / (elements per 128-byte k-block)
  int a_row_end;       // rows >= a_row_end are not stored
  int b_row_end;
  int c_row0, c_col0;  // K[row - c_row0][col - c_col0]
  void* out;
  long long ld;
  int mirror;          // also store the transposed element (symmetric case): 1 = row stores, 2 = TMA store of a transposed tile
  int fix_diag;        // K[g][g] = diag[g] (self similarity over ALL columns)
  int nan_to_num;
  int vec_ok;          // 32-byte aligned rows
  const double* diag;  // self similarity per graph (fp64, exact integers)
  long long* prof;     // optional [gridDim.x][8] cycle counters (GRAKEL_B200_PROF), else NULL
  int tma_store;       // fp32 output through a TMA store of smem-staged 32x32 blocks (tmC valid)
  // multi-GPU row tiling (gk_comm_init): the mirrored half of a tile belongs to the rank that owns K rows
  // [tile.y, tile.y + 256) and is stored straight into THAT rank's row block over NVLink (peer-mapped memory);
  // peer[r] = first row of rank r's block, peer_rows (a multiple of 256) rows per rank.  n_peers = 0: one GPU.
  void* peer[8];
  int n_peers;
  int peer_rows;
  // split-precision GEMM of real-valued features (ShortestPathAttr): k-blocks [k_block0, k_block0 + num_k_blocks) of
  // the panels, result ADDED to `out` when accumulate != 0 (the k range is processed in chunks so that no fp32
  // accumulator sums more than a few hundred MMAs)
  int accumulate;
  int k_block0;
  int k_chunk;         // k-blocks per accumulator (0 = all): the kernel folds every chunk of a tile into `out` itself
  int k_split;         // chunking applies to k-blocks [0, k_split); the rest is ONE chunk (0 = chunk everything)
  const int* nkb_dev;  // number of k-blocks chosen ON THE DEVICE (asynchronous pass, features.cuh GramDyn),
                       // NULL = num_k_blocks
  // Tail fused into the epilogue (TMA-store path with the TMA mirror): the pair updates of the sparse tail, bucketed by
  // 32 x 32 block of K (tail_bucket, features.cuh: tb_cnt[block] entries {row | col << 5 | integer value << 10} at
  // tb_ent[block * TB_CAP ...]), are added to the staged block in shared memory before its bulk store -- instead of a
  // DRAM read-modify-write per update after the GEMM.  NULL = off.
  const unsigned* tb_cnt;
  const unsigned* tb_ent;
  int tb_nb32;         // blocks per row of K
  int tb_cap;          // entries per block the epilogue applies (<= TB_CAP, the storage stride; smaller only in tests)
  int tb_sym;          // 1: only pairs with row < column are bucketed (blocks on or above the block diagonal); a block below
                       // it reads its transpose's list with rows and columns swapped, a diagonal block applies both orders
};
constexpr int TB_CAP = 32;  // entries per block applied in the epilogue (one per lane); the rest go through tb overflow

// tensor maps of the peers' row blocks (multi-GPU, mirrored blocks through TMA: GRAKEL_B200_DIST_TMA)
struct PeerMaps {
  CUtensorMap m[8];
};

// ------------------------------------------------------------------ PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
  } while (!ok);
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int x, int y) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"((unsigned long long)map), "r"(bar), "r"(x), "r"(y)
      : "memory");
}
// the same box written to the same shared-memory offset of every CTA in `mask`; each destination's barrier at
// offset `bar` receives the bytes
__device__ __forceinline__ void tma_load_2d_mc(uint32_t dst, const CUtensorMap* map, uint32_t bar, int x, int y,
                                               uint16_t mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
      " [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(dst), "l"((unsigned long long)map), "r"(bar), "r"(x), "r"(y), "h"(mask)
      : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, uint32_t src, int x, int y) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"((unsigned long long)map), "r"(src), "r"(x), "r"(y)
               : "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// shared::cluster address of `addr` (a shared::cta address of this CTA) in the CTA of rank `rank`
__device__ __forceinline__ uint32_t mapa_u32(uint32_t addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank));
  return r;
}
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t cluster_addr) {
  asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(cluster_addr) : "memory");
}
// barrier of the two warps that stage one 32-row block (ids 1..4; 0 is __syncthreads)
__device__ __forceinline__ void pair_sync(int id) { asm volatile("bar.sync %0, 64;" ::"r"(id) : "memory"); }

// K-major, 128-byte-swizzled shared-memory matrix descriptor of wgmma (one 128-byte row = 64 bf16,
// 128 u8 or 32 tf32 elements; 8-row groups 1024 B apart).  Bit layout: cute::GMMA::GmmaDescriptor.
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFFu) >> 4);  // start address   [0,14)
  d |= (uint64_t)1 << 16;                    // leading byte offset (unused for swizzled K-major)
  d |= (uint64_t)(1024 >> 4) << 32;          // stride byte offset  [32,46)
  d |= (uint64_t)1 << 62;                    // SWIZZLE_128B
  return d;
}

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// accumulator element of each operand kind: s32 for u8 x u8, fp32 otherwise
template <int KIND> struct AccOf { using type = float; };
template <> struct AccOf<2> { using type = int; };

// keeps the compiler from moving accumulator accesses across wgmma fences and waits
__device__ __forceinline__ void acc_fence(float (&d)[128]) {
#pragma unroll
  for (int i = 0; i < 128; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
__device__ __forceinline__ void acc_fence(int (&d)[128]) {
#pragma unroll
  for (int i = 0; i < 128; ++i) asm volatile("" : "+r"(d[i])::"memory");
}

#define GK_F8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), \
                 "+f"(d[i + 6]), "+f"(d[i + 7])
#define GK_F128 GK_F8(0), GK_F8(8), GK_F8(16), GK_F8(24), GK_F8(32), GK_F8(40), GK_F8(48), GK_F8(56), GK_F8(64), \
                GK_F8(72), GK_F8(80), GK_F8(88), GK_F8(96), GK_F8(104), GK_F8(112), GK_F8(120)
#define GK_R8(i) "+r"(d[i]), "+r"(d[i + 1]), "+r"(d[i + 2]), "+r"(d[i + 3]), "+r"(d[i + 4]), "+r"(d[i + 5]), \
                 "+r"(d[i + 6]), "+r"(d[i + 7])
#define GK_R128 GK_R8(0), GK_R8(8), GK_R8(16), GK_R8(24), GK_R8(32), GK_R8(40), GK_R8(48), GK_R8(56), GK_R8(64), \
                GK_R8(72), GK_R8(80), GK_R8(88), GK_R8(96), GK_R8(104), GK_R8(112), GK_R8(120)
#define GK_D128 \
  "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, " \
  "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, "   \
  "%46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, "   \
  "%68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, "   \
  "%90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, "  \
  "%110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}"

// D[64 x 256] (+)= A[64 x k] * B[256 x k]^T, both K-major in shared memory; KIND 0: bf16, k = 16; KIND 1: tf32, k = 8.
// scale_d == 0 overwrites the accumulator.
template <int KIND>
__device__ __forceinline__ void wg_mma(float (&d)[128], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
  if constexpr (KIND == 1)
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k8.f32.tf32.tf32 " GK_D128 ", %128, %129, p, 1, 1;\n\t}"
        : GK_F128
        : "l"(adesc), "l"(bdesc), "r"(scale_d));
  else
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 " GK_D128 ", %128, %129, p, 1, 1, 0, 0;\n\t}"
        : GK_F128
        : "l"(adesc), "l"(bdesc), "r"(scale_d));
}
// KIND 2: u8 x u8 -> s32, k = 32 (integer wgmma has no operand scale or transpose arguments)
template <int KIND>
__device__ __forceinline__ void wg_mma(int (&d)[128], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
  static_assert(KIND == 2, "s32 accumulators belong to the u8 operand kind");
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k32.s32.u8.u8 " GK_D128 ", %128, %129, p;\n\t}"
      : GK_R128
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
}
#undef GK_F8
#undef GK_F128
#undef GK_R8
#undef GK_R128
#undef GK_D128

// Accumulator layout of wgmma m64nN (fp32 or s32): thread `lane` of warp `w` of the warpgroup holds, for every group i of
// 8 columns, d[4i + 2h + e] = D[16 w + lane / 4 + 8 h][8 i + 2 (lane % 4) + e]  (h, e in {0, 1}).

template <typename OutT, bool NORMALIZE>
__device__ __forceinline__ OutT epilogue_value(float acc, int arow, int bcol, double drow, double dcol,
                                               const GramParams& p) {
  if constexpr (NORMALIZE) {
    double v = (double)acc;
    if (p.fix_diag && arow == bcol) v = drow;
    v = v / sqrt(drow * dcol);  // np.divide(K, np.sqrt(np.outer(d, d)))  (fp64, correctly rounded)
    if (p.nan_to_num) {
      if (v != v) v = 0.0;
      else if (isinf(v)) v = v > 0 ? 1.7976931348623157e308 : -1.7976931348623157e308;
    }
    return (OutT)v;
  } else {
    if (p.fix_diag && arow == bcol) return (OutT)drow;
    return (OutT)acc;
  }
}

__device__ __forceinline__ uint32_t swz_addr(uint32_t buf, uint32_t r, uint32_t c) {  // element (r, c) of a staged 32x32 tile
  return buf + r * 128u + ((((c >> 2) ^ (r & 7u))) << 4) + ((c & 3u) << 2);
}

// Epilogue of the 32 x 256 strip [arow0, arow0 + 32) x [tile_y, tile_y + 256) held by one pair of consumer warps
// (`w` = warp in the warpgroup, the pair is w / 2) for fp32, un-normalised output through TMA stores: per 32 x 32
// block, fragments -> 128B-swizzled smem tile -> ONE TMA store (the SM->L2 path is bound by write requests: 1 bulk
// request instead of 32 row stores).  TMA clips at the matrix edge, so partial blocks need no predicates.
template <typename AccT>
__device__ __forceinline__ void epi_tma_store_strip(const GramParams& p, const CUtensorMap* tmC, int arow0, int tile_y,
                                                    const AccT (&acc)[128], int w, int lane, uint32_t my_buf,
                                                    int bar_id, const CUtensorMap* peer_maps) {
  const bool first = (w & 1) == 0;  // the first warp of the pair issues the stores and applies the direct tail list
  const bool leader = first && lane == 0;
  if (arow0 >= p.a_row_end) return;  // uniform over the pair
  const bool diag_tile = p.fix_diag && (arow0 < tile_y + BN) && (tile_y < arow0 + 32);
  const int rb0 = 16 * (w & 1) + (lane >> 2);  // this thread's block rows rb0, rb0 + 8
  float dself[2] = {0.f, 0.f};
  if (diag_tile) {
#pragma unroll
    for (int h = 0; h < 2; ++h)
      if (arow0 + rb0 + 8 * h < p.a_row_end) dself[h] = (float)p.diag[arow0 + rb0 + 8 * h];
  }
  // mirrored rows as plain stores (mirror == 1): K[col][row], in its owner's row block under multi-GPU tiling
  float* mbase = reinterpret_cast<float*>(p.out) + (long long)tile_y * p.ld;
  if (p.n_peers) {
    const int owner = tile_y / p.peer_rows;
    mbase = reinterpret_cast<float*>(p.peer[owner]) + (long long)(tile_y - owner * p.peer_rows) * p.ld;
  }
#pragma unroll
  for (int b = 0; b < BN / 32; ++b) {
    const int bcol0 = tile_y + 32 * b;
    if (bcol0 >= p.b_row_end) break;  // uniform over the pair
    // fused tail: the first warp applies this block's list, the second the mirrored block's
    unsigned tn = 0, te = 0;
    int swap = 0;  // 0: entry as stored, 1: rows and columns swapped, 2: both (diagonal block, symmetric lists)
    if (p.tb_cnt && (first || p.mirror == 2)) {
      const int bx = arow0 >> 5, by = bcol0 >> 5;
      if (p.tb_sym) {  // one list serves the block and its mirror image
        const long long bl = (long long)min(bx, by) * p.tb_nb32 + max(bx, by);
        tn = min(__ldg(&p.tb_cnt[bl]), (unsigned)p.tb_cap);
        te = __ldg(&p.tb_ent[bl * TB_CAP + lane]);
        swap = bx == by ? 2 : ((bx < by) == first ? 0 : 1);
      } else {
        const long long bl = first ? (long long)bx * p.tb_nb32 + by : (long long)by * p.tb_nb32 + bx;
        tn = min(__ldg(&p.tb_cnt[bl]), (unsigned)p.tb_cap);
        te = __ldg(&p.tb_ent[bl * TB_CAP + lane]);
      }
    }
    // buffers: without the TMA mirror the two staging tiles alternate between column blocks; with it tile 0 stages
    // the direct block and tile 1 the transposed one, and both stores of the previous block must have read them
    const uint32_t buf = p.mirror == 2 ? my_buf : my_buf + (uint32_t)(b & 1) * EPI_BUF_BYTES;
    const uint32_t mbuf = my_buf + EPI_BUF_BYTES;
    if (leader) {
      if (p.mirror == 2) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
      else asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
    }
    pair_sync(bar_id);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int rb = rb0 + 8 * h, cb = 8 * j + 2 * (lane & 3);
        float v0 = (float)acc[4 * (4 * b + j) + 2 * h], v1 = (float)acc[4 * (4 * b + j) + 2 * h + 1];
        if (diag_tile) {
          if (arow0 + rb == bcol0 + cb) v0 = dself[h];
          if (arow0 + rb == bcol0 + cb + 1) v1 = dself[h];
        }
        asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(swz_addr(buf, rb, cb)), "f"(v0), "f"(v1) : "memory");
        if (p.mirror == 2) {
          asm volatile("st.shared.f32 [%0], %1;" ::"r"(swz_addr(mbuf, cb, rb)), "f"(v0) : "memory");
          asm volatile("st.shared.f32 [%0], %1;" ::"r"(swz_addr(mbuf, cb + 1, rb)), "f"(v1) : "memory");
        } else if (p.mirror && arow0 + rb < p.a_row_end) {
          float* m = mbase + (long long)(bcol0 + cb - tile_y) * p.ld + arow0 + rb;
          if (bcol0 + cb < p.b_row_end) m[0] = v0;
          if (bcol0 + cb + 1 < p.b_row_end) m[p.ld] = v1;
        }
      }
    }
    pair_sync(bar_id);  // a list entry may land on an element the other warp staged
    if (tn) {  // warp-uniform
      if ((unsigned)lane < tn) {
        const uint32_t e0 = te & 31u, e1 = (te >> 5) & 31u;
        const float val = (float)(te >> 10);
        const uint32_t tb = first ? buf : mbuf;
        if (swap != 1) asm volatile("red.shared.add.f32 [%0], %1;" ::"r"(swz_addr(tb, e0, e1)), "f"(val) : "memory");
        if (swap != 0) asm volatile("red.shared.add.f32 [%0], %1;" ::"r"(swz_addr(tb, e1, e0)), "f"(val) : "memory");
      }
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    pair_sync(bar_id);
    if (leader) {
      tma_store_2d(tmC, buf, bcol0 - p.c_col0, arow0 - p.c_row0);
      if (p.mirror == 2) {
        if (p.n_peers && peer_maps) {  // the block belongs to the rank that owns K rows [bcol0, bcol0 + 32): one bulk store over NVLink
          const int owner = tile_y / p.peer_rows;
          tma_store_2d(&peer_maps[owner], mbuf, arow0, bcol0 - owner * p.peer_rows);
        } else {
          tma_store_2d(tmC, mbuf, arow0 - p.c_col0, bcol0 - p.c_row0);
        }
      }
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    }
  }
  if (leader) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");  // smem reusable by the next tile
}

// Epilogue of the 64 x 256 slab of one consumer warpgroup straight from registers (fp64 output, normalisation,
// split-precision k-chunks that add to `out`, and fp32 output without TMA stores).
template <typename OutT, bool NORMALIZE, typename AccT>
__device__ __forceinline__ void epi_direct(const GramParams& p, int arow_base, int tile_y, const AccT (&acc)[128],
                                           bool acc_out, int lane) {
  OutT* __restrict__ out = reinterpret_cast<OutT*>(p.out);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int arow = arow_base + (lane >> 2) + 8 * h;
    if (arow >= p.a_row_end) continue;
    const double drow = (NORMALIZE || p.fix_diag) ? p.diag[arow] : 0.0;
    OutT* dst_row = out + (long long)(arow - p.c_row0) * p.ld - p.c_col0;
#pragma unroll
    for (int i = 0; i < BN / 8; ++i) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int bcol = tile_y + 8 * i + 2 * (lane & 3) + e;
        if (bcol >= p.b_row_end) continue;
        const double dcol = NORMALIZE ? p.diag[bcol] : 0.0;
        OutT v = epilogue_value<OutT, NORMALIZE>((float)acc[4 * i + 2 * h + e], arow, bcol, drow, dcol, p);
        if (acc_out) v += dst_row[bcol];  // later k-chunks of a split-precision GEMM: this CTA owns the tile
        dst_row[bcol] = v;
        if (p.mirror) out[(long long)bcol * p.ld + arow] = v;
      }
    }
  }
}

// One CTA (PAIR = false: 128 x 256 tiles, B through tmB) or one CTA of a two-CTA cluster (PAIR = true: 256 x 256
// tiles; each CTA computes 128 rows and loads half of the B tile, multicast into both CTAs' shared memory, so the
// pair pulls the B tile from L2 once instead of twice).
template <typename OutT, bool NORMALIZE, int KIND, bool PAIR>
__device__ __forceinline__ void gram_body(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmC,
                                          const GramParams& p, const CUtensorMap* peer_maps) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bar_base = smem_base + STAGES * STAGE_BYTES;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (STAGES + s); };
  const uint32_t epi_base = bar_base + 1024u;  // 1024-byte aligned (128B swizzle atoms)

  const int wgi = threadIdx.x >> 7;
  const uint32_t rank = PAIR ? cluster_ctarank() : 0u;
  const int cid = PAIR ? (int)(blockIdx.x >> 1) : (int)blockIdx.x;
  const int ncl = PAIR ? (int)(gridDim.x >> 1) : (int)gridDim.x;
  const int nkb = p.nkb_dev ? __ldg(p.nkb_dev) : p.num_k_blocks;
  const int kc_base = p.k_chunk > 0 ? p.k_chunk : nkb;
  const int ksplit = p.k_split > 0 ? p.k_split : nkb;

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"((unsigned long long)&tmA) : "memory");
    if (!PAIR) asm volatile("prefetch.tensormap [%0];" ::"l"((unsigned long long)&tmB) : "memory");
    if (p.tma_store) asm volatile("prefetch.tensormap [%0];" ::"l"((unsigned long long)&tmC) : "memory");
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), PAIR ? 16 : 8);  // lane 0 of each consumer warp (of both CTAs of a pair)
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if constexpr (PAIR) cluster_sync_all();  // the peer's barriers are initialised before anything arrives on them

  if (wgi == 0) {
    // registers move from the producer warpgroup to the consumers (128 accumulators each): 40 + 2 x 232 per lane
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (threadIdx.x == 0) {  // ---------------- TMA producer
      int stage = 0;
      uint32_t phase = 0;
      long long w_empty = 0;
      const long long t_start = clock64();
      for (int t = cid; t < p.n_tiles; t += ncl) {
        const int2 tile = p.tiles[t];
        for (int kb = 0; kb < nkb; ++kb) {
          const long long c0 = clock64();
          mbar_wait(empty_bar(stage), phase ^ 1u);
          w_empty += clock64() - c0;
          mbar_expect_tx(full_bar(stage), STAGE_BYTES);
          const uint32_t sa = smem_base + stage * STAGE_BYTES;
          const int kx = (p.k_block0 + kb) * (KIND == 1 ? BK_TF32 : KIND == 2 ? BK_U8 : BK);
          tma_load_2d(sa, &tmA, full_bar(stage), kx, tile.x + (int)rank * BM);
          if constexpr (PAIR)
            tma_load_2d_mc(sa + A_BYTES + rank * (B_BYTES / 2), &tmA, full_bar(stage), kx, tile.y + (int)rank * (BN / 2),
                           (uint16_t)3);
          else
            tma_load_2d(sa + A_BYTES, &tmB, full_bar(stage), kx, tile.y);
          if (++stage == STAGES) { stage = 0; phase ^= 1u; }
        }
      }
      if (p.prof) { p.prof[blockIdx.x * 8 + 5] = w_empty; p.prof[blockIdx.x * 8 + 6] = clock64() - t_start; }
    }
  } else {  // ---------------- consumers: MMA, then the epilogue of their 64 rows
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int wg = wgi - 1;
    const int w = (threadIdx.x >> 5) & 3;
    const int lane = threadIdx.x & 31;
    const uint32_t my_buf = epi_base + (uint32_t)(2 * wg + (w >> 1)) * (2u * EPI_BUF_BYTES);
    const int bar_id = 1 + 2 * wg + (w >> 1);
    const uint32_t peer_rank = rank ^ 1u;
    auto release = [&](int s) {
      if (lane == 0) {
        mbar_arrive(empty_bar(s));
        if constexpr (PAIR) mbar_arrive_cluster(mapa_u32(empty_bar(s), peer_rank));
      }
    };
    typename AccOf<KIND>::type acc[128];
#pragma unroll
    for (int i = 0; i < 128; ++i) acc[i] = 0;
    int stage = 0;
    uint32_t phase = 0;
    long long w_full = 0, t_epi = 0;
    const long long t_start = clock64();
    for (int t = cid; t < p.n_tiles; t += ncl)
    for (int kb0 = 0, kc = 0; kb0 < nkb; kb0 += kc) {  // one accumulator per (tile, k-chunk)
      kc = kb0 < ksplit ? min(kc_base, ksplit - kb0) : nkb - kb0;
      const int kb1 = min(nkb, kb0 + kc);
      int prev = -1;
      for (int kb = kb0; kb < kb1; ++kb) {
        const long long c0 = clock64();
        mbar_wait(full_bar(stage), phase);
        w_full += clock64() - c0;
        const uint32_t sa = smem_base + stage * STAGE_BYTES;
        const uint64_t adesc = wgmma_desc_sw128(sa + (uint32_t)wg * (64u * 128u));
        const uint64_t bdesc = wgmma_desc_sw128(sa + A_BYTES);
        acc_fence(acc);
        wg_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k)  // +32 bytes along K inside the 128-byte swizzle row = +2 in the address field
          wg_mma<KIND>(acc, adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), (uint32_t)((kb - kb0) | k));
        wg_commit();
        wg_wait<1>();  // the previous k-block's MMAs have read their stage
        acc_fence(acc);
        if (prev >= 0) release(prev);
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1u; }
      }
      wg_wait<0>();
      acc_fence(acc);
      if (prev >= 0) release(prev);
      const long long c_e = clock64();
      int2 tile = p.tiles[t];
      tile.x += (int)rank * BM;
      const int arow_slab = tile.x + 64 * wg;
      if (sizeof(OutT) == 4 && !NORMALIZE && p.tma_store)
        epi_tma_store_strip(p, &tmC, arow_slab + 32 * (w >> 1), tile.y, acc, w, lane, my_buf, bar_id, peer_maps);
      else
        epi_direct<OutT, NORMALIZE>(p, arow_slab + 16 * w, tile.y, acc, p.accumulate || kb0 > 0, lane);
      t_epi += clock64() - c_e;
    }
    if (p.prof && threadIdx.x == 128) {
      p.prof[blockIdx.x * 8 + 0] = t_epi; p.prof[blockIdx.x * 8 + 1] = w_full; p.prof[blockIdx.x * 8 + 4] = clock64() - t_start;
    }
    if ((w & 1) == 0 && lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");  // all TMA stores landed
  }
  if constexpr (PAIR) cluster_sync_all();  // neither CTA exits while the peer may still multicast into it or arrive on it
}

template <typename OutT, bool NORMALIZE, int KIND = 0 /* 0: bf16 operands, 1: tf32 operands, 2: u8 operands */>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gram_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               const __grid_constant__ CUtensorMap tmC, GramParams p) {
  gram_body<OutT, NORMALIZE, KIND, false>(tmA, tmB, tmC, p, nullptr);
}

// ---------------------------------------------------------------------------
// Exact CUDA-core Gram over a u32 count panel (int64 accumulation).  Used (a) as
// the on-device cross-check of the tensor-core kernel in the tests and (b) when a
// count exceeds 256 or a Gram value exceeds 2^24, where neither operand type of the
// tensor-core kernel holds the counts or fp32 no longer holds the result exactly.
template <typename OutT, bool NORMALIZE>
__global__ void __launch_bounds__(256)
gram_simt_kernel(const unsigned* __restrict__ panel, long long ldp, int kdim, int a_row0, int a_row_end,
                 int b_row0, int b_row_end, GramParams p) {
  __shared__ unsigned As[16][17], Bs[16][17];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int arow = a_row0 + blockIdx.y * 16 + ty;
  const int bcol = b_row0 + blockIdx.x * 16 + tx;
  unsigned long long acc = 0;
  for (int k0 = 0; k0 < kdim; k0 += 16) {
    const int ar = a_row0 + blockIdx.y * 16 + ty;
    const int br = b_row0 + blockIdx.x * 16 + ty;
    As[ty][tx] = (ar < a_row_end && k0 + tx < kdim) ? panel[(long long)ar * ldp + k0 + tx] : 0u;
    Bs[ty][tx] = (br < b_row_end && k0 + tx < kdim) ? panel[(long long)br * ldp + k0 + tx] : 0u;
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 16; ++k) acc += (unsigned long long)As[ty][k] * Bs[tx][k];
    __syncthreads();
  }
  if (arow >= a_row_end || bcol >= b_row_end) return;
  double v = (double)acc;
  const double drow = p.diag[arow], dcol = p.diag[bcol];
  if (p.fix_diag && arow == bcol) v = drow;
  if (NORMALIZE) {
    v = v / sqrt(drow * dcol);
    if (p.nan_to_num) {
      if (v != v) v = 0.0;
      else if (isinf(v)) v = v > 0 ? 1.7976931348623157e308 : -1.7976931348623157e308;
    }
  }
  reinterpret_cast<OutT*>(p.out)[(long long)(arow - p.c_row0) * p.ld + (bcol - p.c_col0)] = (OutT)v;
}

// K with no contracted columns: zero matrix (+ exact diagonal / normalisation)
template <typename OutT, bool NORMALIZE>
__global__ void __launch_bounds__(256)
gram_empty_kernel(int a_row0, int a_row_end, int b_row0, int b_row_end, GramParams p) {
  const long long n_cols = b_row_end - b_row0;
  const long long total = (long long)(a_row_end - a_row0) * n_cols;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int arow = a_row0 + (int)(i / n_cols), bcol = b_row0 + (int)(i % n_cols);
    double v = 0.0;
    const double drow = p.diag[arow], dcol = p.diag[bcol];
    if (p.fix_diag && arow == bcol) v = drow;
    if (NORMALIZE) {
      v = v / sqrt(drow * dcol);
      if (p.nan_to_num) {
        if (v != v) v = 0.0;
        else if (isinf(v)) v = v > 0 ? 1.7976931348623157e308 : -1.7976931348623157e308;
      }
    }
    reinterpret_cast<OutT*>(p.out)[(long long)(arow - p.c_row0) * p.ld + (bcol - p.c_col0)] = (OutT)v;
  }
}

}  // namespace gk
