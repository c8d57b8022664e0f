// Jagged HSTU attention forward on the wgmma kernels when the value head is wider than the query / key head: dqk < dv, both
// in {32, 64, 128, 256}, bf16 / fp16, full attention and delta-q (attn_wgmma_fwd.cuh, DESIGN.md 3.7).  S = Q K^T reduces
// over dqk and O += P V has N = dv; the O accumulator is dv / 2 registers per thread, so (32, 64) runs two CTAs per SM like
// d = 64, and the pairs with dv >= 128 one.  Every pair has a 3-stage K / V ring.  bf16 inputs keep the hi / lo split of P
// at dqk = 32 too: the scaled fp16 pre-pass of attn_fp16_operands.cu is a dqk == dv == 32 feature.
#include "attn_wgmma_fwd.cuh"

namespace hstu {

template <int DQK, int DV, bool BF16>
__global__ void __launch_bounds__(kAttnThreads, kFwdMinBlocks<DV>) attn_fwd_mixed_wgmma_kernel(const __grid_constant__ FwdParams p) {
  attn_fwd_wgmma_body<DQK, DV, BF16, false>(p);
}
template <int DQK, int DV, bool BF16>
__global__ void __launch_bounds__(kAttnThreads, kFwdMinBlocks<DV>) attn_fwd_delta_mixed_wgmma_kernel(const __grid_constant__ FwdParams p) {
  attn_fwd_wgmma_body<DQK, DV, BF16, true>(p);
}

int attn_wgmma_fwd_mixed(const hstu_attn_params& p, cudaStream_t st) {
  return dispatch_dims(MixedDims{}, p, "wgmma forward", [&]<int DQK, int DV, bool BF16>() {
    if (p.delta_q_len > 0) return launch_fwd_wgmma<DQK, DV, BF16, true>(p, st, attn_fwd_delta_mixed_wgmma_kernel<DQK, DV, BF16>);
    return launch_fwd_wgmma<DQK, DV, BF16, false>(p, st, attn_fwd_mixed_wgmma_kernel<DQK, DV, BF16>);
  });
}

}  // namespace hstu
