// Non-causal (bidirectional) jagged HSTU attention on the wgmma kernels at dqk == dv in {32, 64, 128} (bf16 / fp16): the
// forward, the split dK / dV and dQ backward, their support check and their routing (DESIGN.md 3.9).
//
// The kernels are the causal ones' bodies (attn_wgmma_fwd.cuh, attn_wgmma_bwd.cuh) instantiated with kBidir: the key range
// of a query tile and the query range of a key tile come from the non-causal ranges of common.cuh, and each tile takes one
// of the mask cases of mask_scores_bidir.  Everything else -- the K / V ring, the TMA / mbarrier pipeline, the MMAs, the
// epilogues, the scaled fp16 operands of bf16 at d = 32 (DESIGN.md 3.0) -- is the causal kernels' own code.  They have
// names of their own so that the causal kernels stay the only instances of theirs.
// The backward is the atomic-free split pair at every head dim: one backward, bitwise reproducible, with no workspace
// beyond the fp16 operands of bf16 at d = 32.
#include "attn_wgmma_bwd.cuh"
#include "attn_wgmma_fwd.cuh"

namespace hstu {

template <int D, bool BF16>
__global__ void __launch_bounds__(kAttnThreads, kFwdMinBlocks<D>) attn_fwd_bidir_wgmma_kernel(const __grid_constant__ FwdParams p) {
  attn_fwd_wgmma_body<D, D, BF16, false, true>(p);
}

template <int D, bool BF16>
__global__ void __launch_bounds__(kAttnThreads, split_min_blocks(D)) attn_bwd_dkdv_bidir_wgmma_kernel(const __grid_constant__ BwdParams p) {
  bwd_key_tile<D, D, BF16, false, true>(p);
}

template <int D, bool BF16>
__global__ void __launch_bounds__(kAttnThreads, split_min_blocks(D)) attn_bwd_dq_bidir_wgmma_kernel(const __grid_constant__ BwdParams p) {
  bwd_dq_body<D, D, BF16, true>(p);
}

using BidirDims = HeadDimList<HeadDims<32, 32>, HeadDims<64, 64>, HeadDims<128, 128>>;

bool wgmma_bidir_supported(const hstu_attn_params& p, bool bwd) {
  return p.delta_q_len == 0 && has_dims(BidirDims{}, p.dqk, p.dv) && wgmma_supported(p, bwd);
}

size_t wgmma_bidir_workspace_bytes(const hstu_attn_params& p, bool bwd) {
  return runs_on_fp16_operands(p) ? fp16_operands_workspace_bytes(p, bwd) : 0;
}

int attn_wgmma_bidir_fwd(const hstu_attn_params& p, cudaStream_t st) {
  return dispatch_dims(BidirDims{}, p, "non-causal wgmma forward", [&]<int D, int, bool BF16>() {
    if constexpr (scaled_fp16_dims(BF16, D, D)) {  // the fp16 kernel on exactly scaled copies (DESIGN.md 3.0)
      Fp16Operands f16;
      if (int e = fp16_operands_prepass(p, false, &f16, st)) return e;
      return launch_fwd_wgmma<D, D, false, false>(p, st, attn_fwd_bidir_wgmma_kernel<D, false>, &f16);
    } else {
      return launch_fwd_wgmma<D, D, BF16, false>(p, st, attn_fwd_bidir_wgmma_kernel<D, BF16>);
    }
  });
}

int attn_wgmma_bidir_bwd(const hstu_attn_params& p, cudaStream_t st) {
  return dispatch_dims(BidirDims{}, p, "non-causal wgmma backward", [&]<int D, int, bool BF16>() {
    if constexpr (scaled_fp16_dims(BF16, D, D)) {
      Fp16Operands f16;
      if (int e = fp16_operands_prepass(p, true, &f16, st)) return e;
      return launch_bwd_split<D, D, false>(p, st, attn_bwd_dkdv_bidir_wgmma_kernel<D, false>, attn_bwd_dq_bidir_wgmma_kernel<D, false>,
                                           &f16);
    } else {
      return launch_bwd_split<D, D, BF16>(p, st, attn_bwd_dkdv_bidir_wgmma_kernel<D, BF16>, attn_bwd_dq_bidir_wgmma_kernel<D, BF16>);
    }
  });
}

}  // namespace hstu
