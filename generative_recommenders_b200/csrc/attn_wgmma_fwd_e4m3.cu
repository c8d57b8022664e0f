// Jagged HSTU attention forward on float8 e4m3 q, k, v with per (sequence, head) descales, bf16 output, on the Hopper
// warpgroup tensor cores, at dqk == dv in {32, 64, 128, 256}; the host checks and routing of every fp8 forward.  The kernel
// body, its design and its launcher are in attn_wgmma_fwd_e4m3.cuh; the dqk < dv instantiations are in
// attn_wgmma_mixed_fwd_e4m3.cu (DESIGN.md 3.5).
#include "attn_wgmma_fwd_e4m3.cuh"

namespace hstu {

template <int D>
__global__ void __launch_bounds__(kAttnThreads, kE4m3MinBlocks<D>) attn_fwd_e4m3_wgmma_kernel(const __grid_constant__ E4m3FwdParams p) {
  attn_fwd_e4m3_body<D, D>(p);
}

// ------------------------------------------------------------------------------------------------
// host
// ------------------------------------------------------------------------------------------------
// fp8 views: 16-byte base, and row / head strides of whole 16-byte units (TMA strides and the pre-pass's 8-byte loads)
bool e4m3_view(const void* ptr, long long row_stride, long long head_stride) {
  return (reinterpret_cast<uintptr_t>(ptr) & 15) == 0 && (row_stride % 16) == 0 && (head_stride % 16) == 0;
}

int e4m3_fwd_check(const hstu_attn_params& p) {
  if (!wgmma_dims(p.dqk, p.dv)) {
    set_error("fp8 attention: dqk == dv or dqk < dv, both in {32, 64, 128, 256}, only (dqk=%d, dv=%d)", p.dqk, p.dv);
    return HSTU_ERR_UNSUPPORTED;
  }
  if (p.delta_q_len != 0 || p.pos_w != nullptr || p.ts_w != nullptr) {
    set_error("fp8 attention: delta_q and the relative bias are not supported");
    return HSTU_ERR_UNSUPPORTED;
  }
  if (p.total_rows >= (1ll << 31) - 256) {
    set_error("fp8 attention: at most 2^31 - 257 rows (got %lld)", (long long)p.total_rows);
    return HSTU_ERR_UNSUPPORTED;
  }
  if (!e4m3_view(p.q, p.q_row_stride, p.q_head_stride) || !e4m3_view(p.k, p.k_row_stride, p.k_head_stride) ||
      !e4m3_view(p.v, p.v_row_stride, p.v_head_stride)) {
    set_error("fp8 attention: q, k, v need 16-byte aligned bases and row / head strides that are multiples of 16 elements");
    return HSTU_ERR_UNSUPPORTED;
  }
  if (!aligned_view(p.out, p.o_row_stride, p.o_head_stride)) {
    set_error("fp8 attention: out needs a 16-byte aligned base and row / head strides that are multiples of 8 elements");
    return HSTU_ERR_UNSUPPORTED;
  }
  return 0;
}

int attn_wgmma_fwd_e4m3(const hstu_attn_params& p, const hstu_attn_descales& ds, cudaStream_t st) {
  if (int e = e4m3_fwd_check(p)) return e;
  const void* v16 = nullptr;
  if (int e = e4m3_v_prepass(p, &v16, st)) return e;
  if (p.dqk != p.dv) return attn_wgmma_fwd_e4m3_mixed(p, ds, v16, st);
  return dispatch_dims(SquareDims{}, p, "fp8 attention", [&]<int D, int, bool>() {
    return launch_fwd_e4m3<D, D>(p, ds, v16, st, attn_fwd_e4m3_wgmma_kernel<D>);
  });
}

}  // namespace hstu
