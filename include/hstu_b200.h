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
 *   hstu_attn_fwd_bidir / hstu_attn_bwd_bidir (causal=False)
 *        ops/hstu_attention.py:44-128 hstu_mha(causal=False); ops/pytorch/pt_hstu_attention.py:33-84 (the mask)
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

/* HSTU_E4M3: float8 e4m3fn q, k, v of hstu_attn_fwd_fp8 only (its output is bf16); every other entry point rejects it. */
typedef enum hstu_dtype { HSTU_F32 = 0, HSTU_BF16 = 1, HSTU_F16 = 2, HSTU_E4M3 = 3 } hstu_dtype;

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
  HSTU_IMPL_UMMA = 2   /* force wgmma + TMA kernels (bf16/fp16, dqk == dv in {32, 64, 128, 256}, delta_q included;
                          backward up to 128) */
} hstu_attn_impl;

/* One jagged attention problem: q,k [L, H, dqk], v [L, H, dv], last-dim stride 1, arbitrary row and head
 * strides (in elements) -- q/k/v may be views into one fused `uvqk` buffer.  Sequence b owns rows
 * [seq_offsets[b], seq_offsets[b+1]).  Semantics: pt_hstu_attention.py:130-171 (see DESIGN.md).          */
typedef struct hstu_attn_params {
  int32_t abi_version;  /* = HSTU_B200_ABI_VERSION */
  int32_t dtype;        /* hstu_dtype of q,k,v,out,dout,dq,dk,dv (HSTU_E4M3: of q,k,v; out is bf16) */
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
  int32_t delta_q_len;  /* 0 = full attention; > 0: q is [B*delta_q_len, H, dqk], the last rows of each sequence (forward
                           only; keys are every row of the sequence, not clipped to max_seq_len).  On the wgmma path the
                           keys may be split into chunks whose fp32 partials need hstu_attn_workspace_bytes() of scratch */
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
/* bf16 / fp16 / fp32 attention; HSTU_E4M3 inputs go through hstu_attn_fwd_fp8 (and have no backward). */
int hstu_attn_fwd(const hstu_attn_params* p, void* cuda_stream);
int hstu_attn_bwd(const hstu_attn_params* p, void* cuda_stream);

/* A bf16 attention at dqk == dv == 32 runs on the wgmma kernels on exactly scaled fp16 copies of q, k, v (and dO) with their
 * per (sequence, head) amax, which a pre-pass writes before each call.  A forward can leave its copies to the caller, and
 * the backward of the same q, k, v (same seq_offsets, max_seq_len and alpha) can then take them instead: it scales and
 * converts dO alone.  dq, dk, dv are bitwise those of hstu_attn_bwd.
 * hstu_attn_fp16_operands_bytes: bytes of the caller's operands buffer ([B, H, 4] amax bits, then the fp16 copies of q, k
 * and v, [L, H, 32] each), or 0 if the call does not run on such operands (another dtype or head dim, delta_q, a relative
 * bias, the generic kernels) or is empty.
 * hstu_attn_fwd_keep_fp16_operands: hstu_attn_fwd writing them into `operands` (operands_bytes >= that many, 256-byte
 * aligned); it uses no workspace.  HSTU_ERR_UNSUPPORTED where hstu_attn_fp16_operands_bytes is 0.
 * hstu_attn_bwd_on_fp16_operands: hstu_attn_bwd on such a buffer of operands_bytes bytes, unchanged since its forward
 * (HSTU_ERR_INVALID_ARGUMENT if it is smaller than these sizes need); q, k, v and their strides are not read (they may be
 * NULL / 0).  dout, dq, dk, dv must be views the wgmma backward takes (16-byte base, row / head strides of whole 16-byte
 * units): there is no generic fallback without q, k, v.  Its workspace: hstu_attn_bwd_fp16_operands_workspace_bytes(p)
 * bytes (dO's amax and copy; sizes only). */
size_t hstu_attn_fp16_operands_bytes(const hstu_attn_params* p);
int hstu_attn_fwd_keep_fp16_operands(const hstu_attn_params* p, void* operands, size_t operands_bytes, void* cuda_stream);
size_t hstu_attn_bwd_fp16_operands_workspace_bytes(const hstu_attn_params* p);
int hstu_attn_bwd_on_fp16_operands(const hstu_attn_params* p, const void* operands, size_t operands_bytes,
                                   void* cuda_stream);

/* Per (sequence, head) dequantisation scales of the fp8 forward.  Each pointer is an fp32 device array read at
 * [b * batch_stride + h * head_stride] (strides in elements, >= 0), or NULL for a scale of 1. */
typedef struct hstu_attn_descales {
  const float* q;
  const float* k;
  const float* v;
  int64_t q_batch_stride, q_head_stride;
  int64_t k_batch_stride, k_head_stride;
  int64_t v_batch_stride, v_head_stride;
} hstu_attn_descales;
/* Forward of fp8 attention (the reference's e4m3 forward, flash_api.cpp hstu_mha_fwd with q/k/v_descale): p->dtype is
 * HSTU_E4M3 and out is bf16; out = attention(q * q_descale[b, h], k * k_descale[b, h], v * v_descale[b, h]) with every
 * mask option of hstu_attn_fwd.  wgmma kernels only (sm_90): dqk == dv, or dqk < dv, with both in {32, 64, 128, 256}
 * (out has dv columns), no delta_q, no relative bias; q / k / v bases 16-byte aligned with row and head strides that are
 * multiples of 16 elements.  Other shapes (dqk > dv among them) return HSTU_ERR_UNSUPPORTED.  Needs a workspace of
 * hstu_attn_workspace_bytes(p, 0) bytes (an fp16 copy of v, L * H * dv * 2 rounded up to 256).
 * descales may be NULL (all scales 1). */
int hstu_attn_fwd_fp8(const hstu_attn_params* p, const hstu_attn_descales* descales, void* cuda_stream);
/* KV-cached (delta-q) forward with 16-bit queries over an fp8 K / V cache: p->dtype (HSTU_BF16 or HSTU_F16) is the type
 * of q and out, k and v are float8 e4m3fn, and out = delta_attention(q, k * k_descale[b, h], v * v_descale[b, h]) with
 * every mask option of hstu_attn_fwd.  descales->q must be NULL; descales, or its k / v, may be NULL (scale 1).  wgmma
 * kernels only (sm_90, p->impl other than HSTU_IMPL_GENERIC): delta_q_len > 0, no relative bias, dqk == dv or dqk < dv
 * with both in {32, 64, 128, 256}; q and out 16-byte aligned with row / head strides that are multiples of 8 elements, k
 * and v 16-byte aligned with multiples of 16.  Anything else returns HSTU_ERR_UNSUPPORTED.  When the keys are split into
 * chunks it needs a workspace of hstu_attn_fp8_kv_workspace_bytes(p) bytes (the fp32 partials, the rule of the 16-bit
 * delta-q forward).  hstu_attn_select_impl and hstu_attn_workspace_bytes do not describe this entry. */
int hstu_attn_fwd_delta_fp8_kv(const hstu_attn_params* p, const hstu_attn_descales* descales, void* cuda_stream);
/* Workspace of hstu_attn_fwd_delta_fp8_kv (sizes only, no device query): 0 with one key chunk or a call it refuses. */
size_t hstu_attn_fp8_kv_workspace_bytes(const hstu_attn_params* p);
/* Which implementation a call would dispatch to: returns HSTU_IMPL_GENERIC or HSTU_IMPL_UMMA (<0 on error).  A
 * deterministic backward returns HSTU_IMPL_UMMA where the wgmma backward supports the shape (it then runs its atomic-free
 * dK / dV and dQ kernels), else HSTU_IMPL_GENERIC; HSTU_ERR_UNSUPPORTED with a relative bias, or with impl forced to
 * HSTU_IMPL_UMMA on a shape the wgmma backward does not support.  For HSTU_E4M3 the answer depends on the shape only (the
 * workspace size must be computable without a device): HSTU_IMPL_UMMA where the fp8 forward takes the shape, whatever the
 * device, and hstu_attn_fwd_fp8 itself then returns HSTU_ERR_UNSUPPORTED on a device other than sm_90. */
int hstu_attn_select_impl(const hstu_attn_params* p, int is_backward);

/* Non-causal (causal=False) attention: hstu_attn_fwd / hstu_attn_bwd under the reference eager path's causal=False mask
 * (pt_hstu_attention.py:33-84): with the ids of the causal mask, dist = |id_i - id_j|, valid = (i == j) | (dist > 0), then
 * max_attn_len / min_full_attn_seq_len on dist and the contextual rule.  History rows see the target keys; a target row
 * sees every history key (within the window) and of the target keys only its own.  Same params and semantics otherwise
 * (alpha, 1 / max_seq_len, rows >= max_seq_len zero).  HSTU_ERR_UNSUPPORTED for delta_q_len > 0, a relative bias or
 * HSTU_E4M3.  The wgmma kernels take bf16 / fp16 at dqk == dv in {32, 64, 128} (the backward: atomic-free dK / dV and dQ
 * kernels at every dim, so it is bitwise reproducible whatever `deterministic` says); everything else runs the generic
 * kernels.  hstu_attn_bidir_select_impl / hstu_attn_bidir_workspace_bytes answer as hstu_attn_select_impl /
 * hstu_attn_workspace_bytes do for the causal calls. */
int hstu_attn_fwd_bidir(const hstu_attn_params* p, void* cuda_stream);
int hstu_attn_bwd_bidir(const hstu_attn_params* p, void* cuda_stream);
size_t hstu_attn_bidir_workspace_bytes(const hstu_attn_params* p, int is_backward);
int hstu_attn_bidir_select_impl(const hstu_attn_params* p, int is_backward);

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

/* The same under the non-causal mask (hstu_attn_fwd_bidir).  Without max_attn_len both ranges are [0, len). */
int hstu_mask_valid_bidir(int32_t len, int32_t num_targets, int32_t max_attn_len, int32_t min_full_attn_seq_len,
                          int32_t contextual_seq_len, int32_t i, int32_t j);
int hstu_kv_range_for_q_rows_bidir(int32_t len, int32_t num_targets, int32_t max_attn_len, int32_t min_full_attn_seq_len,
                                   int32_t contextual_seq_len, int32_t m0, int32_t m1, int32_t* lo, int32_t* hi);
int hstu_q_range_for_kv_rows_bidir(int32_t len, int32_t num_targets, int32_t max_attn_len, int32_t min_full_attn_seq_len,
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
 * out [L, N]; fp32 accumulation, result in `dtype`.  Every row is written, however long its sequence: rows at positions
 * >= max_seq_len of a sequence are exact zeros (the eager path truncates at max_seq_len and pads those rows with 0).          */
int hstu_jagged_dense_bmm_broadcast_add(const void* jagged, const void* dense, const void* bias, void* out,
                                        const void* seq_offsets, int32_t offsets_are_i64, int32_t batch, int32_t K, int32_t N,
                                        int32_t max_seq_len, int32_t dense_is_transposed, int32_t dtype, void* cuda_stream);
/* d_dense[b] = jagged[rows of b]^T @ dout[rows of b]  ([B, K, N]);  d_bias[b] = sum of dout rows of b ([B, N], nullable);
 * only the rows at positions < max_seq_len of each sequence take part, as in the forward.                                   */
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
