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

template <int DQK, int DV>
static int launch_mixed(const hstu_attn_params& p, cudaStream_t st) {
  if (p.dtype == HSTU_BF16)
    return launch_bwd_split<DQK, DV, true>(p, st, attn_bwd_dkdv_mixed_wgmma_kernel<DQK, DV, true>,
                                           attn_bwd_dq_mixed_wgmma_kernel<DQK, DV, true>);
  return launch_bwd_split<DQK, DV, false>(p, st, attn_bwd_dkdv_mixed_wgmma_kernel<DQK, DV, false>,
                                          attn_bwd_dq_mixed_wgmma_kernel<DQK, DV, false>);
}

int attn_wgmma_bwd_mixed(const hstu_attn_params& p, cudaStream_t st) {
  switch (p.dqk * 1000 + p.dv) {
    case 32064: return launch_mixed<32, 64>(p, st);
    case 32128: return launch_mixed<32, 128>(p, st);
    case 32256: return launch_mixed<32, 256>(p, st);
    case 64128: return launch_mixed<64, 128>(p, st);
    case 64256: return launch_mixed<64, 256>(p, st);
    case 128256: return launch_mixed<128, 256>(p, st);
  }
  set_error("wgmma backward: unsupported head dims dqk = %d, dv = %d", p.dqk, p.dv);
  return HSTU_ERR_UNSUPPORTED;
}

}  // namespace hstu
