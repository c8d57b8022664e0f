// Jagged HSTU attention forward on float8 e4m3 q, k, v when the value head is wider than the query / key head: dqk < dv,
// both in {32, 64, 128, 256}, bf16 output (attn_wgmma_fwd_e4m3.cuh, DESIGN.md 3.5).  S = Q K^T reduces over dqk on the fp8
// tensor cores, and its P exponent bound takes dqk; O += P' V has N = dv on the fp16 copy of v.  The O accumulator is dv / 2
// registers per thread, so (32, 64) runs two CTAs per SM with the merged MMA batch, like d = 64, and the pairs with dv >= 128
// one CTA per SM without it.  Every pair has a 3-stage K / V ring: 136 KB of shared memory at (128, 256).
#include "attn_wgmma_fwd_e4m3.cuh"

namespace hstu {

template <int DQK, int DV>
__global__ void __launch_bounds__(kAttnThreads, kE4m3MinBlocks<DV>) attn_fwd_e4m3_mixed_wgmma_kernel(const __grid_constant__ E4m3FwdParams p) {
  attn_fwd_e4m3_body<DQK, DV>(p);
}

int attn_wgmma_fwd_e4m3_mixed(const hstu_attn_params& p, const hstu_attn_descales& ds, const void* v16, cudaStream_t st) {
  return dispatch_dims(MixedDims{}, p, "fp8 attention", [&]<int DQK, int DV, bool>() {
    return launch_fwd_e4m3<DQK, DV>(p, ds, v16, st, attn_fwd_e4m3_mixed_wgmma_kernel<DQK, DV>);
  });
}

}  // namespace hstu
