/*
 * hstu_b200.h -- C ABI of libhstu_b200.so: the H100 (sm_90a) backend of the HSTU hot path.
 *
 * Every entry point takes raw device pointers, element strides and sizes -- no ATen / torch types cross
 * this boundary.  All functions return 0 on success and a negative code on failure; the message is
 * available through hstu_last_error() (thread-local).  Kernels are enqueued on the caller's stream and
 * the library never synchronises the device.
 *
 * Reference interfaces each entry point replaces (paths under
 * generative_recommenders/ of the reference):
 *
 *   hstu_attn_fwd / hstu_attn_bwd
 *        ops/hstu_attention.py:44-128            hstu_mha (python facade, kernel=HammerKernel.CUDA)
 *        ops/hstu_attention.py:131-203           delta_hstu_mha (params.delta_q_len > 0)
 *        ops/cpp/hstu_attention/flash_api.cpp:275-352  hstu::hstu_mha_fwd / hstu::hstu_mha_bwd schemas
 *        ops/cpp/hstu_attention/flash.h:23-134   Flash_fwd_params / Flash_bwd_params (field meaning)
 *        research/modeling/sequential/hstu.py:150-223  attention with relative bias (params.pos_w != NULL)
 *   hstu_layer_norm_fwd / _bwd, hstu_rms_norm_fwd / _bwd
 *        ops/layer_norm.py:46-184, ops/pytorch/pt_layer_norm.py:24-61, ops/triton/triton_layer_norm.py
 *   hstu_norm_mul_dropout_fwd / _bwd
 *        ops/pytorch/pt_hstu_linear.py:23-66, ops/triton/triton_hstu_linear.py:48-1036
 *   hstu_silu_fwd / _bwd
 *        ops/hstu_compute.py:86 (u = silu(u)) and its autograd
 *   hstu_jagged_concat / hstu_jagged_split
 *        ops/jagged_tensors.py:55-207, ops/pytorch/pt_jagged_tensors.py:31-246,
 *        ops/triton/triton_jagged_tensors.py:31-142
 *   hstu_position_embeddings_fwd / _bwd
 *        ops/position.py:43-96, ops/pytorch/pt_position.py:39-134, ops/triton/triton_position.py:58-435
 *   hstu_jagged_dense_bmm_broadcast_add / hstu_jagged_dense_bmm_wgrad
 *        ops/jagged_tensors.py:210-253, ops/pytorch/pt_jagged.py:77-98, ops/triton/triton_jagged.py:56-347
 *   hstu_sampled_softmax_fwd / _bwd
 *        research/modeling/sequential/losses/sampled_softmax.py:29-193, autoregressive_losses.py:73-121
 *   hstu_mask_valid / hstu_kv_tile_range (host-side helpers, no GPU needed)
 *        ops/pytorch/pt_hstu_attention.py:33-84 (_get_valid_attn_mask)
 */
#ifndef HSTU_B200_H_
#define HSTU_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define HSTU_B200_ABI_VERSION 1

typedef enum hstu_dtype { HSTU_F32 = 0, HSTU_BF16 = 1, HSTU_F16 = 2 } hstu_dtype;

typedef enum hstu_status {
  HSTU_OK = 0,
  HSTU_ERR_INVALID_ARGUMENT = -1,
  HSTU_ERR_UNSUPPORTED = -2,
  HSTU_ERR_CUDA = -3,
  HSTU_ERR_WORKSPACE = -4
} hstu_status;

/* Every implementation honours hstu_attn_params.deterministic: with it set, AUTO runs the backward on the atomic-free
 * wgmma kernels where the shape allows (bf16/fp16, dqk == dv in {32, 64, 128}) and on the generic kernels otherwise. */
typedef enum hstu_attn_impl {
  HSTU_IMPL_AUTO = 0,  /* wgmma/TMA kernels when the shape allows, else the generic kernels */
  HSTU_IMPL_GENERIC = 1, /* CUDA-core fp32-accumulate kernels: any dtype / head dim <= 256 / all mask options */
  HSTU_IMPL_UMMA = 2   /* force wgmma + TMA kernels (bf16/fp16, dqk == dv in {32, 64, 128, 256}; backward up to 128) */
} hstu_attn_impl;

/* One jagged attention problem: q,k [L, H, dqk], v [L, H, dv], last-dim stride 1, arbitrary row and head
 * strides (in elements) -- q/k/v may be views into one fused `uvqk` buffer.  Sequence b owns rows
 * [seq_offsets[b], seq_offsets[b+1]).  Semantics: pt_hstu_attention.py:130-171 (see DESIGN.md).          */
typedef struct hstu_attn_params {
  int32_t abi_version;  /* = HSTU_B200_ABI_VERSION */
  int32_t dtype;        /* hstu_dtype of q,k,v,out,dout,dq,dk,dv */
  int32_t impl;         /* hstu_attn_impl */
  int32_t batch;        /* B */
  int32_t heads;        /* H */
  int32_t dqk;          /* attention dim */
  int32_t dv;           /* hidden / linear dim per head */
  int32_t max_seq_len;  /* N: scores are divided by N, rows >= N of a sequence are ignored */
  int64_t total_rows;   /* L = seq_offsets[B] (rows of k,v; rows of q unless delta_q_len > 0) */
  float alpha;
  int32_t max_attn_len;           /* 0 = unlimited */
  int32_t min_full_attn_seq_len;  /* only used when max_attn_len > 0 */
  int32_t contextual_seq_len;
  int32_t delta_q_len;  /* 0 = full attention; > 0: q is [B*delta_q_len, H, dqk], the last rows of each sequence */
  int32_t offsets_are_i64;      /* seq_offsets element type: 0 = int32, 1 = int64 */
  int32_t num_targets_are_i64;  /* num_targets element type */
  const void* seq_offsets;      /* [B+1] device */
  const void* num_targets;      /* [B] device or NULL */
  const void* q;
  const void* k;
  const void* v;
  void* out;             /* [Lq, H, dv] */
  int64_t q_row_stride, q_head_stride;
  int64_t k_row_stride, k_head_stride;
  int64_t v_row_stride, v_head_stride;
  int64_t o_row_stride, o_head_stride;
  /* backward only */
  const void* dout;
  void* dq;
  void* dk;
  void* dv_out;
  int64_t do_row_stride, do_head_stride;
  int64_t dq_row_stride, dq_head_stride;
  int64_t dk_row_stride, dk_head_stride;
  int64_t dv_row_stride, dv_head_stride;
  /* optional relative bias (research path): S += pos_w[n-1+j-i] + ts_w[bucket(ts[i+1]-ts[j])]; alpha applies to QK^T only */
  const float* pos_w;        /* [2*max_seq_len-1] or NULL */
  const float* ts_w;         /* [num_ts_buckets+1] or NULL */
  const int64_t* timestamps; /* [B, max_seq_len] or NULL */
  int32_t num_ts_buckets;
  int32_t deterministic;     /* backward: 0 = fastest kernels (d = 64 / 128 on wgmma add dQ with fp32 atomics);
                                1 = dq / dk / dv bitwise reproducible run to run (no relative bias: HSTU_ERR_UNSUPPORTED) */
  float* dpos_w;             /* backward: fp32 accumulators (atomically added), or NULL */
  float* dts_w;
  /* scratch */
  void* workspace;           /* >= hstu_attn_workspace_bytes() bytes, 256-byte aligned, or NULL if 0 */
  size_t workspace_bytes;
} hstu_attn_params;

const char* hstu_last_error(void);
int hstu_abi_version(void);

/* Bytes of scratch the call needs (is_backward: 0 fwd, 1 bwd).  Depends only on sizes/dtype/impl/deterministic. */
size_t hstu_attn_workspace_bytes(const hstu_attn_params* p, int is_backward);
int hstu_attn_fwd(const hstu_attn_params* p, void* cuda_stream);
int hstu_attn_bwd(const hstu_attn_params* p, void* cuda_stream);
/* Which implementation a call would dispatch to: returns HSTU_IMPL_GENERIC or HSTU_IMPL_UMMA (<0 on error).  A
 * deterministic backward returns HSTU_IMPL_UMMA where the wgmma backward supports the shape (it then runs its atomic-free
 * dK / dV and dQ kernels), else HSTU_IMPL_GENERIC; HSTU_ERR_UNSUPPORTED with a relative bias, or with impl forced to
 * HSTU_IMPL_UMMA on a shape the wgmma backward does not support. */
int hstu_attn_select_impl(const hstu_attn_params* p, int is_backward);

/* ---- host-side helpers (pure CPU; used by the no-GPU tests to pin the mask / tile-skipping logic) ---- */
/* 1 if query position i may attend key position j (both < len) -- pt_hstu_attention.py:33-84. */
int hstu_mask_valid(int32_t len, int32_t num_targets /* <0: none */, int32_t max_attn_len,
                    int32_t min_full_attn_seq_len, int32_t contextual_seq_len, int32_t i, int32_t j);
/* Conservative key range [lo, hi) that query rows [m0, m1) can attend (what the kernels iterate over). */
int hstu_kv_range_for_q_rows(int32_t len, int32_t num_targets, int32_t max_attn_len, int32_t min_full_attn_seq_len,
                             int32_t contextual_seq_len, int32_t m0, int32_t m1, int32_t* lo, int32_t* hi);
/* Conservative query range [lo, hi) (plus the contextual prefix [0, ctx_hi)) attending keys [n0, n1). */
int hstu_q_range_for_kv_rows(int32_t len, int32_t num_targets, int32_t max_attn_len, int32_t min_full_attn_seq_len,
                             int32_t contextual_seq_len, int32_t n0, int32_t n1, int32_t* lo, int32_t* hi,
                             int32_t* ctx_hi);

/* ---- row-wise normalisation (HBM-bound) ---- */
/* y = LN(x) * w + b (w,b nullable); swish != 0: y = x * sigmoid(LN(x)*w+b).  mean/rstd [n_rows] fp32 saved for bwd
 * (nullable).  x,y rows have D contiguous elements and row strides x_row_stride / y_row_stride.           */
int hstu_layer_norm_fwd(const void* x, const void* w, const void* b, void* y, float* mean, float* rstd,
                        int64_t n_rows, int32_t D, int64_t x_row_stride, int64_t y_row_stride, float eps,
                        int32_t dtype, int32_t swish, void* cuda_stream);
/* dx (and fp32 dw, db [D], nullable) from dy; recomputes xhat from x, mean, rstd.  partial: fp32 scratch of
 * hstu_norm_bwd_partial_rows() * 2 * D floats used for the two-stage dw/db reduction.                     */
int hstu_layer_norm_bwd(const void* dy, const void* x, const void* w, const void* b, const float* mean,
                        const float* rstd, void* dx, float* dw, float* db, float* partial, int64_t n_rows,
                        int32_t D, int64_t x_row_stride, int64_t dy_row_stride, int64_t dx_row_stride,
                        int32_t dtype, int32_t swish, void* cuda_stream);
int32_t hstu_norm_bwd_partial_rows(void);
/* RMSNorm: y = x * rsqrt(mean(x^2)+eps) * w  (ops/layer_norm.py:138-158). */
int hstu_rms_norm_fwd(const void* x, const void* w, void* y, float* rstd, int64_t n_rows, int32_t D, float eps,
                      int32_t dtype, void* cuda_stream);
int hstu_rms_norm_bwd(const void* dy, const void* x, const void* w, const float* rstd, void* dx, float* dw,
                      float* partial, int64_t n_rows, int32_t D, int32_t dtype, void* cuda_stream);

/* Output stage (pt_hstu_linear.py:23-66): y = u' * Norm(attn) with u' = silu_u ? silu(u) : u; Norm = LayerNorm over
 * all H*dv columns (group_norm=0, w,b [H*dv]) or per-head GroupNorm (group_norm=1, w,b [H]).
 * concat_ux: 1: out row = [u' | attn | y] (3*H*dv wide); 2: [u' | Norm(attn) | y] (the research block's concat_ua,
 * research/modeling/sequential/hstu.py:427-430); 0: [y].  Dropout with keep-prob 1-p uses a counter-based
 * generator keyed by (seed, element index); p = 0 is exact.  mean/rstd: [n_rows * (group_norm ? H : 1)].  */
int hstu_norm_mul_dropout_fwd(const void* attn, const void* u, const void* w, const void* b, void* out, float* mean,
                              float* rstd, int64_t n_rows, int32_t heads, int32_t dv, int64_t attn_row_stride,
                              int64_t u_row_stride, float eps, float dropout_p, uint64_t seed, int32_t dtype,
                              int32_t silu_u, int32_t concat_ux, int32_t group_norm, void* cuda_stream);
int hstu_norm_mul_dropout_bwd(const void* dout, const void* attn, const void* u, const void* w, const void* b,
                              const float* mean, const float* rstd, void* dattn, void* du, float* dw, float* db,
                              float* partial, int64_t n_rows, int32_t heads, int32_t dv, int64_t attn_row_stride,
                              int64_t u_row_stride, int64_t dattn_row_stride, int64_t du_row_stride, float dropout_p,
                              uint64_t seed, int32_t dtype, int32_t silu_u, int32_t concat_ux, int32_t group_norm,
                              void* cuda_stream);

/* y = silu(x) over [n_rows, n_cols] with row strides (in place allowed); dx = dy * dsilu(x). */
int hstu_silu_fwd(const void* x, void* y, int64_t n_rows, int32_t n_cols, int64_t x_row_stride, int64_t y_row_stride,
                  int32_t dtype, void* cuda_stream);
int hstu_silu_bwd(const void* dy, const void* x, void* dx, int64_t n_rows, int32_t n_cols, int64_t dy_row_stride,
                  int64_t x_row_stride, int64_t dx_row_stride, int32_t dtype, void* cuda_stream);

/* Jagged concat / split of [rows, D] matrices (verbatim row copies; routing is integer-exact):
 *   out_b = [ right_b[:n_prefix] | left_b | right_b[n_prefix:] ]
 * offsets_left / offsets_right: [B+1] device (int32 or int64 per offsets_are_i64) or NULL for a dense side with
 * dense_len_left / dense_len_right rows per batch entry.  split is the inverse (writes left and right).     */
int hstu_jagged_concat(const void* left, const void* right, void* out, const void* offsets_left,
                       const void* offsets_right, int32_t offsets_are_i64, int32_t batch, int32_t dense_len_left,
                       int32_t dense_len_right, int32_t n_prefix, int32_t D, int32_t elem_bytes, int32_t max_seq_len,
                       void* cuda_stream);
int hstu_jagged_split(const void* in, void* left, void* right, const void* offsets_left, const void* offsets_right,
                      int32_t offsets_are_i64, int32_t batch, int32_t dense_len_left, int32_t dense_len_right,
                      int32_t n_prefix, int32_t D, int32_t elem_bytes, int32_t max_seq_len, void* cuda_stream);

/* Timestamp + position embedding add in front of the STU stack (ops/position.py:43-96, ops/pytorch/pt_position.py:39-134):
 *   out[r] = cast(seq[r] * alpha) + cast(pos_w[pos_ind(r)] + ts_w[ts_bucket(r)])       (tables fp32, activations `dtype`)
 * pos_ind / ts_bucket as the eager code computes them (see csrc/position.cu); they are also written to pos_inds / ts_inds
 * ([total_rows] int32, nullable) for the backward.  timestamps: [total_rows] int64 (jagged).  num_time_buckets is the clamp
 * the caller wants (the eager path uses ts_w.size(1) - 1).  log_time_bucket: 1 = log, 0 = sqrt.                        */
int hstu_position_embeddings_fwd(const void* seq_embeddings, void* out, const float* pos_w, const float* ts_w,
                                 const void* seq_offsets, const void* seq_lengths, const void* num_targets,
                                 const int64_t* timestamps, int32_t* pos_inds, int32_t* ts_inds, int64_t total_rows,
                                 int32_t batch, int32_t D, int32_t max_pos_ind, int32_t num_time_buckets,
                                 int32_t max_contextual_seq_len, float alpha, int32_t interleave_targets,
                                 int32_t log_time_bucket, int32_t offsets_are_i64, int32_t lengths_are_i64,
                                 int32_t num_targets_are_i64, int32_t dtype, void* cuda_stream);
/* d_seq = dout * alpha; d_pos_w[pos_inds[r]] += dout[r]; d_ts_w[ts_inds[r]] += dout[r] (fp32 tables, zero-initialised by the
 * caller, accumulated with atomics).                                                                                     */
int hstu_position_embeddings_bwd(const void* dout, void* d_seq_embeddings, float* d_pos_w, float* d_ts_w,
                                 const int32_t* pos_inds, const int32_t* ts_inds, int64_t total_rows, int32_t D, float alpha,
                                 int32_t dtype, void* cuda_stream);

/* out[rows of sequence b] = jagged[rows of b] @ dense[b] + bias[b]  (ops/jagged_tensors.py:210-253, ops/pytorch/pt_jagged.py:77-98):
 * jagged [L, K], dense [B, K, N] (or [B, N, K] with dense_is_transposed: the d_jagged = dout @ dense^T pass), bias [B, N] or NULL,
 * out [L, N]; fp32 accumulation, result in `dtype`.  Rows at positions >= max_seq_len of a sequence are written as zeros.     */
int hstu_jagged_dense_bmm_broadcast_add(const void* jagged, const void* dense, const void* bias, void* out,
                                        const void* seq_offsets, int32_t offsets_are_i64, int32_t batch, int32_t K, int32_t N,
                                        int32_t max_seq_len, int32_t dense_is_transposed, int32_t dtype, void* cuda_stream);
/* d_dense[b] = jagged[rows of b]^T @ dout[rows of b]  ([B, K, N]);  d_bias[b] = sum of dout rows of b ([B, N], nullable).      */
int hstu_jagged_dense_bmm_wgrad(const void* jagged, const void* dout, void* d_dense, void* d_bias, const void* seq_offsets,
                                int32_t offsets_are_i64, int32_t batch, int32_t K, int32_t N, int32_t max_seq_len, int32_t dtype,
                                void* cuda_stream);

/* Fused sampled-softmax loss with dot-product similarity over negatives gathered straight from the item embedding table
 * (research/modeling/sequential/losses/sampled_softmax.py:43-89; LocalNegativesSampler autoregressive_losses.py:73-121;
 * dot_product_similarity_fn.py:31-67).  Row i: logits = [q_i . n(pos_emb_i), q_i . n(table[neg_ids[i, r]]) ...] / T with
 * n(x) = x / max(||x||, l2_eps) if l2_norm; negatives whose id equals pos_ids[i] get -5e4; loss_rows[i] = lse_i - logits[i, 0].
 * The weighted mean over rows is left to the caller.  D must be (16 / sizeof(dtype)) * 2^k, 2^k <= 32.                     */
typedef struct hstu_ssl_params {
  int32_t abi_version;  /* = HSTU_B200_ABI_VERSION */
  int32_t dtype;        /* hstu_dtype of q, pos_emb, table, d_q, d_pos_emb */
  int64_t N;            /* query rows */
  int32_t R;            /* negatives per row */
  int32_t D;            /* embedding dim */
  int32_t l2_norm;
  float l2_eps;
  float temperature;
  int32_t reserved0;
  const void* q;            /* [N, D] */
  const void* pos_emb;      /* [N, D] (before normalisation) */
  const void* table;        /* [V, D] item embedding table */
  const int64_t* pos_ids;   /* [N] */
  const int64_t* neg_ids;   /* [N, R], every id < V */
  float* logits;            /* [N, R + 1] fwd out / bwd in (column 0 = positive) */
  float* rnorm;             /* [N, R + 1] fwd out / bwd in: 1 / max(||e||, eps) (1 without l2_norm) */
  float* lse;               /* [N] fwd out / bwd in */
  float* loss_rows;         /* [N] fwd out */
  const float* row_coef;    /* [N] bwd in: dloss * w_i / sum(w) */
  void* d_q;                /* [N, D] bwd out */
  void* d_pos_emb;          /* [N, D] bwd out, zero-initialised by the caller */
  float* d_table;           /* [V, D] fp32 bwd out, zero-initialised by the caller (atomically accumulated) */
} hstu_ssl_params;
int hstu_sampled_softmax_fwd(const hstu_ssl_params* p, void* cuda_stream);
int hstu_sampled_softmax_bwd(const hstu_ssl_params* p, void* cuda_stream);

#ifdef __cplusplus
}
#endif
#endif /* HSTU_B200_H_ */
