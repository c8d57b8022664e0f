// Jagged HSTU attention backward on the wgmma kernels when the value head is wider than the query / key head: dqk < dv, both
// in {32, 64, 128, 256}, bf16 / fp16 (attn_wgmma_bwd.cuh, DESIGN.md 3.7).  Always the two split kernels, with no atomics and
// no workspace; a deterministic backward at these dims stays on the generic kernels (wgmma_bwd_supported).
//   dK / dV (bwd_key_tile): S^T reduces over dqk and dP^T over dv.  At dv = 256 two CTAs share a key tile, one half of the dK
//                           and of the dV columns each ((128, 256): 32 + 64 accumulator registers per thread), on 32-row
//                           query tiles; every pair has a 4-stage Q_j / dO_j ring.
//   dQ (bwd_dq_body):       Q (dqk) and dO (dv) resident, K and V streamed, the dQ accumulator dqk wide; 64-key tiles,
//                           32 at (128, 256), in a 3-stage ring.
// bf16 inputs keep the hi / lo split of P and dS at dqk = 32 too: the scaled fp16 pre-pass is a dqk == dv == 32 feature.
#include "attn_wgmma_bwd.cuh"

namespace hstu {

template <int DQK, int DV, bool BF16>
__global__ void __launch_bounds__(kAttnThreads, split_min_blocks(DV)) attn_bwd_dkdv_mixed_wgmma_kernel(const __grid_constant__ BwdParams p) {
  bwd_key_tile<DQK, DV, BF16, false>(p);
}
template <int DQK, int DV, bool BF16>
__global__ void __launch_bounds__(kAttnThreads, split_min_blocks(DV)) attn_bwd_dq_mixed_wgmma_kernel(const __grid_constant__ BwdParams p) {
  bwd_dq_body<DQK, DV, BF16>(p);
}

int attn_wgmma_bwd_mixed(const hstu_attn_params& p, cudaStream_t st) {
  return dispatch_dims(MixedDims{}, p, "wgmma backward", [&]<int DQK, int DV, bool BF16>() {
    return launch_bwd_split<DQK, DV, BF16>(p, st, attn_bwd_dkdv_mixed_wgmma_kernel<DQK, DV, BF16>,
                                           attn_bwd_dq_mixed_wgmma_kernel<DQK, DV, BF16>);
  });
}

}  // namespace hstu
