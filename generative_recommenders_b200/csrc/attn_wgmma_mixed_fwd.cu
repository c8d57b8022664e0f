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

template <int DQK, int DV, bool BF16>
static int launch_mixed(const hstu_attn_params& p, cudaStream_t st) {
  if (p.delta_q_len > 0) return launch_fwd_wgmma<DQK, DV, BF16, true>(p, st, attn_fwd_delta_mixed_wgmma_kernel<DQK, DV, BF16>);
  return launch_fwd_wgmma<DQK, DV, BF16, false>(p, st, attn_fwd_mixed_wgmma_kernel<DQK, DV, BF16>);
}
template <int DQK, int DV>
static int launch_mixed(const hstu_attn_params& p, cudaStream_t st) {
  return p.dtype == HSTU_BF16 ? launch_mixed<DQK, DV, true>(p, st) : launch_mixed<DQK, DV, false>(p, st);
}

int attn_wgmma_fwd_mixed(const hstu_attn_params& p, cudaStream_t st) {
  switch (p.dqk * 1000 + p.dv) {
    case 32064: return launch_mixed<32, 64>(p, st);
    case 32128: return launch_mixed<32, 128>(p, st);
    case 32256: return launch_mixed<32, 256>(p, st);
    case 64128: return launch_mixed<64, 128>(p, st);
    case 64256: return launch_mixed<64, 256>(p, st);
    case 128256: return launch_mixed<128, 256>(p, st);
  }
  set_error("wgmma forward: unsupported head dims dqk = %d, dv = %d", p.dqk, p.dv);
  return HSTU_ERR_UNSUPPORTED;
}

}  // namespace hstu
