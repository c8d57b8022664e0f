// Internal (non-ABI) declarations shared by the translation units of libhstu_b200.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#include "../../include/hstu_b200.h"

namespace hstu {
void set_error(const char* fmt, ...);

// attn_generic.cu (bidir: the non-causal mask of common.cuh)
int attn_generic_fwd(const hstu_attn_params& p, cudaStream_t st, bool bidir = false);
int attn_generic_bwd(const hstu_attn_params& p, cudaStream_t st, bool bidir = false);

// The head dims of the wgmma attention kernels: dqk == dv, or dqk < dv, both in {32, 64, 128, 256}.  attn_wgmma_fwd.cu,
// attn_wgmma_bwd.cu and attn_wgmma_fwd_e4m3.cu instantiate the square pairs, the attn_wgmma_mixed_*.cu units the others.
template <int DQK, int DV> struct HeadDims {};
template <class... Pairs> struct HeadDimList {};
using SquareDims = HeadDimList<HeadDims<32, 32>, HeadDims<64, 64>, HeadDims<128, 128>, HeadDims<256, 256>>;
using MixedDims = HeadDimList<HeadDims<32, 64>, HeadDims<32, 128>, HeadDims<32, 256>, HeadDims<64, 128>, HeadDims<64, 256>,
                              HeadDims<128, 256>>;
// The non-causal kernels (attn_wgmma_bidir.cu) instantiate dqk == dv in {32, 64, 128} only.
using BidirDims = HeadDimList<HeadDims<32, 32>, HeadDims<64, 64>, HeadDims<128, 128>>;
template <int... DQK, int... DV>
constexpr bool has_dims(HeadDimList<HeadDims<DQK, DV>...>, int dqk, int dv) { return ((dqk == DQK && dv == DV) || ...); }
inline bool wgmma_dims(int dqk, int dv) { return has_dims(SquareDims{}, dqk, dv) || has_dims(MixedDims{}, dqk, dv); }

// f.template operator()<DQK, DV, BF16>() for the pair of `dims` that is (p.dqk, p.dv), with BF16 = (p.dtype == HSTU_BF16);
// HSTU_ERR_UNSUPPORTED if there is none
template <int... DQK, int... DV, class F>
int dispatch_dims(HeadDimList<HeadDims<DQK, DV>...>, const hstu_attn_params& p, const char* what, F&& f) {
  int rc = HSTU_ERR_UNSUPPORTED;
  const bool bf = p.dtype == HSTU_BF16;
  const bool found = ((p.dqk == DQK && p.dv == DV &&
                       (rc = bf ? f.template operator()<DQK, DV, true>() : f.template operator()<DQK, DV, false>(), true)) || ...);
  if (!found) set_error("%s: unsupported head dims dqk = %d, dv = %d", what, p.dqk, p.dv);
  return rc;
}

// bf16 at dqk == dv == 32 runs the fp16 kernels on exactly scaled copies of its operands (attn_fp16_operands.cu,
// DESIGN.md 3.0), except in the delta-q forward, which keeps the bf16 kernel.  The wgmma units instantiate no other bf16
// kernel at these dims.
constexpr bool scaled_fp16_dims(bool bf16, int dqk, int dv) { return bf16 && dqk == 32 && dv == 32; }
inline bool runs_on_fp16_operands(const hstu_attn_params& p) {
  return scaled_fp16_dims(p.dtype == HSTU_BF16, p.dqk, p.dv) && p.delta_q_len == 0;
}
// The fused backward kernel (dK, dV and dQ atomics into an fp32 workspace) exists at d = 64 and 128.  The backward splits
// into atomic-free dK / dV and dQ kernels at every other dim, at dqk < dv, and when it must be deterministic (DESIGN.md
// 3.2); at d = 256 the fused kernel's fp32 dQ accumulator would be L * H * 1 KB.
constexpr bool fused_bwd_dims(int dqk, int dv) { return dqk == dv && (dqk == 64 || dqk == 128); }
inline bool split_dq(const hstu_attn_params& p) { return !fused_bwd_dims(p.dqk, p.dv) || p.deterministic != 0; }

// attn_wgmma_fwd.cu: whether the wgmma kernels take the call (dtype, dims, bias, views; sm_90; bidir: the non-causal mask,
// BidirDims and no delta-q) and the forward; attn_wgmma_bwd.cu: the workspace and the backward
bool wgmma_supported(const hstu_attn_params& p, bool bwd, bool bidir);
size_t wgmma_workspace_bytes(const hstu_attn_params& p, bool bwd, bool bidir);
int attn_wgmma_fwd(const hstu_attn_params& p, cudaStream_t st);
int attn_wgmma_bwd(const hstu_attn_params& p, cudaStream_t st);
// attn_wgmma_bidir.cu: the non-causal forward and its (split) backward
int attn_wgmma_bidir_fwd(const hstu_attn_params& p, cudaStream_t st);
int attn_wgmma_bidir_bwd(const hstu_attn_params& p, cudaStream_t st);
// attn_wgmma_bwd.cu: the bf16 d = 32 backward on the fp16 operands a forward kept (hstu_attn_bwd_on_fp16_operands)
int attn_wgmma_bwd_on_fp16_operands(const hstu_attn_params& p, const void* kept, cudaStream_t st);
// attn_wgmma_mixed_fwd.cu / attn_wgmma_mixed_bwd.cu: the same at dqk < dv (both in {32, 64, 128, 256})
int attn_wgmma_fwd_mixed(const hstu_attn_params& p, cudaStream_t st);
int attn_wgmma_bwd_mixed(const hstu_attn_params& p, cudaStream_t st);
// attn_wgmma_fwd.cu: a 16-bit view the kernels take (16-byte base, row / head strides of whole 16-byte units)
bool aligned_view(const void* ptr, long long row_stride, long long head_stride);
// the delta-q forward's fp32 partials of its key chunks (0 when one chunk suffices); sizes only
size_t wgmma_delta_workspace_bytes(const hstu_attn_params& p);

// attn_fp16_operands.cu: per (sequence, head) amax and exactly scaled fp16 copies of the bf16 d = 32 operands
struct Fp16Operands {
  const unsigned int* amax;  // [B, H, 4] bits of max |q|, |k|, |v|, |dO| (attn_fp16_operands.cuh)
  const void* copy[4];       // fp16 [L, H, 32] copies of q, k, v, dO (dO: backward only)
};
size_t fp16_operands_workspace_bytes(const hstu_attn_params& p, bool bwd);
// the amax block at the start of `buf` (a workspace, or the operands buffer of a kept-operands call) and the copies after it
// (as many as `buf` holds)
Fp16Operands fp16_operands_at(const hstu_attn_params& p, void* buf);
int fp16_operands_prepass(const hstu_attn_params& p, bool bwd, Fp16Operands* out, cudaStream_t st);
// the backward on operands a forward kept (hstu_attn_bwd_on_fp16_operands): q, k, v and their amax from `kept`, dO's amax
// and copy into the workspace
size_t fp16_operands_dout_workspace_bytes(const hstu_attn_params& p);
int fp16_operands_dout_prepass(const hstu_attn_params& p, const void* kept, Fp16Operands* out, cudaStream_t st);
// the fp8 forward's fp16 copy of the e4m3 v, [L, H, dv] contiguous (exact: no scale), at the start of the workspace
size_t e4m3_v_copy_bytes(const hstu_attn_params& p);
int e4m3_v_prepass(const hstu_attn_params& p, const void** v16, cudaStream_t st);

// attn_wgmma_fwd_e4m3.cu: the fp8 forward.  e4m3_fwd_check: 0 if the wgmma fp8 kernels take the shape (sizes, flags and
// alignment only, no device query), else HSTU_ERR_UNSUPPORTED with a message
int e4m3_fwd_check(const hstu_attn_params& p);
int attn_wgmma_fwd_e4m3(const hstu_attn_params& p, const hstu_attn_descales& ds, cudaStream_t st);
// attn_wgmma_mixed_fwd_e4m3.cu: its dqk < dv kernels, on the fp16 copy v16 of v that attn_wgmma_fwd_e4m3 has written
int attn_wgmma_fwd_e4m3_mixed(const hstu_attn_params& p, const hstu_attn_descales& ds, const void* v16, cudaStream_t st);
// attn_wgmma_fwd_e4m3.cu: an e4m3 view the kernels take (16-byte base, row / head strides of whole 16-byte units)
bool e4m3_view(const void* ptr, long long row_stride, long long head_stride);
bool is_sm90();

// attn_wgmma_delta_fp8kv.cu: the delta-q forward with 16-bit q and out over an e4m3 K / V cache (DESIGN.md 3.8).
// delta_fp8_kv_check: 0 if its kernels take the call (dtype, delta, bias, impl, dims, row limits, views; no device query),
// else HSTU_ERR_UNSUPPORTED with a message
int delta_fp8_kv_check(const hstu_attn_params& p);
int attn_wgmma_fwd_delta_fp8_kv(const hstu_attn_params& p, const hstu_attn_descales& ds, cudaStream_t st);

// norm.cu
int layer_norm_fwd(const void* x, const void* w, const void* b, void* y, float* mean, float* rstd, long long n, int D,
                   long long xs, long long ys, float eps, int dtype, int swish, bool rms, cudaStream_t st);
int layer_norm_bwd(const void* dy, const void* x, const void* w, const void* b, const float* mean, const float* rstd,
                   void* dx, float* dw, float* db, float* partial, long long n, int D, long long xs, long long dys,
                   long long dxs, int dtype, int swish, bool rms, cudaStream_t st);
int norm_mul_dropout_fwd(const void* attn, const void* u, const void* w, const void* b, void* out, float* mean,
                         float* rstd, long long n, int H, int dv, long long as, long long us, float eps, float p,
                         unsigned long long seed, int dtype, int silu_u, int concat, int gn, cudaStream_t st);
int norm_mul_dropout_bwd(const void* dout, const void* attn, const void* u, const void* w, const void* b,
                         const float* mean, const float* rstd, void* dattn, void* du, float* dw, float* db,
                         float* partial, long long n, int H, int dv, long long as, long long us, long long das,
                         long long dus, float p, unsigned long long seed, int dtype, int silu_u, int concat, int gn,
                         cudaStream_t st);
int silu_fwd_bwd(const void* x, const void* dy, void* out, long long n, int cols, long long xs, long long dys,
                 long long os, int dtype, bool bwd, cudaStream_t st);
int norm_partial_rows();

// position.cu
struct PosArgs {
  const void* seq;      // [L, D] activation dtype
  void* out;            // [L, D]
  const float* pos_w;   // [max_pos_ind, D] fp32
  const float* ts_w;    // [ts_rows, D] fp32
  const void* seq_offsets;   // [B+1]
  const void* seq_lengths;   // [B]
  const void* num_targets;   // [B] or NULL
  const long long* timestamps;  // [L] int64
  int* pos_inds;        // [L] out (saved for backward) or NULL
  int* ts_inds;         // [L] out or NULL
  long long L;
  int B, D;
  int max_pos_ind, num_time_buckets, max_contextual;
  int offsets_i64, lengths_i64, targets_i64;
  int interleave, log_bucket, vec_ok;
  float alpha;
};
int position_fwd(const PosArgs& a, int dtype, cudaStream_t st);
int position_bwd(const void* dout, void* dseq, float* dpos, float* dts, const int* pos_inds, const int* ts_inds, long long L, int D,
                 float alpha, int dtype, cudaStream_t st);

// sampled_softmax.cu
typedef hstu_ssl_params SslArgs;
int sampled_softmax_fwd(const SslArgs& a, int dtype, cudaStream_t st);
int sampled_softmax_bwd(const SslArgs& a, int dtype, cudaStream_t st);

// jagged_bmm.cu
int jagged_bmm(const void* A, const void* Bm, const void* bias, void* C, const void* off, int off_i64, int batch, int K, int N,
               int max_seq_len, bool trans_b, int dtype, cudaStream_t st);
int jagged_bmm_wgrad(const void* A, const void* G, void* dW, void* dbias, const void* off, int off_i64, int batch, int K, int N,
                     int max_seq_len, int dtype, cudaStream_t st);

// jagged.cu
int jagged_concat_split(bool split, const void* a, const void* b, void* c, void* c2, const void* off_l, const void* off_r,
                        int is_i64, int batch, int dense_l, int dense_r, int n_prefix, int D, int elem_bytes,
                        int max_seq_len, cudaStream_t st);
}  // namespace hstu
