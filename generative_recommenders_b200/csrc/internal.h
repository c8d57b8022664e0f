// Internal (non-ABI) declarations shared by the translation units of libhstu_b200.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#include "../../include/hstu_b200.h"

namespace hstu {
void set_error(const char* fmt, ...);

// attn_generic.cu
int attn_generic_fwd(const hstu_attn_params& p, cudaStream_t st);
int attn_generic_bwd(const hstu_attn_params& p, cudaStream_t st);

// attn_wgmma_fwd.cu / attn_wgmma_bwd.cu
bool wgmma_supported(const hstu_attn_params& p, bool bwd);
size_t wgmma_workspace_bytes(const hstu_attn_params& p, bool bwd);
int attn_wgmma_fwd(const hstu_attn_params& p, cudaStream_t st);
int attn_wgmma_bwd(const hstu_attn_params& p, cudaStream_t st);

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
