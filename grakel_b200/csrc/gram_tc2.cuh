// Cluster-pair variant of the Gram GEMM: one 256 x 256 output tile per cluster of two CTAs, fp32 un-normalised
// output through the TMA-store epilogue of gram_tc.cuh.
//
// Why: the B tile (256 panel rows) is the same for both 128-row halves of a 256 x 256 tile.  Each CTA of the pair
// loads its own 128 rows of A and HALF of the B tile, multicast into both CTAs' shared memory: 32 KB pulled from L2
// per CTA and k-block instead of 48 KB for the same flops.
//
// Protocol (same shared-memory offsets in both CTAs):
//   full[s]   (one per CTA)  1 arrival (the CTA's own arrive.expect_tx of 48 KB): its A load, its B half and the
//             peer's multicast B half complete their bytes on it
//   empty[s]  (one per CTA)  16 arrivals: lane 0 of the eight consumer warps of EACH CTA (the peer's through mapa),
//             because the CTA's next load of stage s writes into both CTAs' shared memory
//
// KIND 0: bf16 panel (f32 accumulators), KIND 2: u8 panel (s32 accumulators); the k-block is 128 bytes either way.
#pragma once
#include "gram_tc.cuh"

namespace gk {

constexpr int BM2 = 256;  // rows of A per cluster tile (128 per CTA)
constexpr int GEMM2_SMEM = GEMM_SMEM;

template <int KIND>
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(GEMM_THREADS, 1)
gram_tc2_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmC, GramParams p,
                const __grid_constant__ PeerMaps pm) {
  gram_body<float, false, KIND, true>(tmA, tmA, tmC, p, p.mirror == 2 && p.n_peers ? pm.m : nullptr);
}

}  // namespace gk
