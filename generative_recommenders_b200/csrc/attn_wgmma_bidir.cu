// Non-causal (bidirectional) jagged HSTU attention on the wgmma kernels at dqk == dv in {32, 64, 128} (bf16 / fp16): the
// forward and the split dK / dV and dQ backward (DESIGN.md 3.9).  Which calls they take (the bidir case of wgmma_supported)
// and their workspace (of wgmma_workspace_bytes) are decided with the causal kernels' own.
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

int attn_wgmma_bidir_fwd(const hstu_attn_params& p, cudaStream_t st) {
  return dispatch_dims(BidirDims{}, p, "non-causal wgmma forward", [&]<int D, int, bool BF16>() {
    return launch_on_operands<D, BF16>(p, false, st, [&]<bool B>(const Fp16Operands* f16) {
      return launch_fwd_wgmma<D, D, B, false>(p, st, attn_fwd_bidir_wgmma_kernel<D, B>, f16);
    });
  });
}

int attn_wgmma_bidir_bwd(const hstu_attn_params& p, cudaStream_t st) {
  return dispatch_dims(BidirDims{}, p, "non-causal wgmma backward", [&]<int D, int, bool BF16>() {
    return launch_on_operands<D, BF16>(p, true, st, [&]<bool B>(const Fp16Operands* f16) {
      return launch_bwd_split<D, D, B>(p, st, attn_bwd_dkdv_bidir_wgmma_kernel<D, B>, attn_bwd_dq_bidir_wgmma_kernel<D, B>, f16);
    });
  });
}

}  // namespace hstu
