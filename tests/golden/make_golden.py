"""Generate golden vectors from the UNMODIFIED reference eager path.

    python tests/golden/make_golden.py   # checkout at /root/reference, or HSTU_REFERENCE_ROOT=<checkout>; writes tests/golden/*.pt

The reference ships no golden vectors for the HSTU hot path (SURVEY.md section 8c); these fixtures are
outputs of the reference's own PyTorch-eager code (generative_recommenders @ 2e81fab, imported from
a checkout of it) on seeded inputs, with the three fbgemm_gpu jagged ops supplied by
oracle/fbgemm_shim.py.  They pin the CPU oracle (tests/test_oracle_vs_golden.py) and, through it and
directly, the CUDA kernels (tests/test_gpu_*.py).  The tests need no checkout of the reference: only
these committed fixtures.
"""
import os
import random
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
REF_ROOT = os.environ.get("HSTU_REFERENCE_ROOT") or "/root/reference"
if not os.path.isdir(os.path.join(REF_ROOT, "generative_recommenders")):
    sys.exit(f"make_golden.py: no checkout of generative-recommenders at {REF_ROOT} (set HSTU_REFERENCE_ROOT)")
sys.path.insert(0, REF_ROOT)

from oracle import fbgemm_shim  # noqa: E402

fbgemm_shim.install()

import torch  # noqa: E402
from generative_recommenders.common import HammerKernel  # noqa: E402
from generative_recommenders.modules.stu import STULayer, STULayerConfig, STUStack  # noqa: E402
from generative_recommenders.ops.hstu_attention import delta_hstu_mha, hstu_mha  # noqa: E402
from generative_recommenders.ops.hstu_compute import hstu_compute_output  # noqa: E402
from generative_recommenders.ops.jagged_tensors import (  # noqa: E402
    concat_2D_jagged,
    hstu_concat_l2_embeddings,
    hstu_split_l2_embeddings,
    split_2D_jagged,
)
from generative_recommenders.ops.layer_norm import layer_norm, swish_layer_norm  # noqa: E402

PT = HammerKernel.PYTORCH


def offsets_from(lengths):
    off = torch.zeros(len(lengths) + 1, dtype=torch.int64)
    off[1:] = torch.cumsum(torch.as_tensor(lengths, dtype=torch.int64), 0)
    return off


def attn_case(name, seed, B, H, max_uih, max_tgt, dqk, dv, targets, max_attn_len, ctx, min_full, dtype):
    # input recipe of ops/tests/hstu_attention_test.py:60-102
    g = torch.Generator().manual_seed(seed)
    lengths = torch.randint(max_uih + 1, (B,), generator=g)
    lengths[0] = 0 if B > 2 else lengths[0]  # force an empty-history sequence
    nt = torch.randint(1, max_tgt + 1, (B,), generator=g)
    lengths = lengths + nt + ctx
    N = max_uih + max_tgt + ctx
    off = offsets_from(lengths.tolist())
    L = int(off[-1])
    mk = lambda d: torch.empty(L, H, d).uniform_(-0.1, 0.1, generator=g).to(dtype)  # noqa: E731
    q, k, v = mk(dqk), mk(dqk), mk(dv)
    dout = torch.randn(L, H, dv, generator=g).to(dtype)
    alpha = 1.0 / dqk**0.5
    res = {}
    for tag, cd in (("f32", torch.float32), ("native", dtype)):
        qq, kk, vv = (t.to(cd).clone().requires_grad_() for t in (q, k, v))
        out = hstu_mha(
            max_seq_len=N, alpha=alpha, q=qq, k=kk, v=vv, seq_offsets=off, causal=True,
            num_targets=nt if targets else None, max_attn_len=max_attn_len, contextual_seq_len=ctx,
            min_full_attn_seq_len=min_full, kernel=PT,
        )
        out.backward(dout.to(cd))
        res[tag] = dict(out=out.detach(), dq=qq.grad, dk=kk.grad, dv=vv.grad)
    torch.save(
        dict(
            name=name, max_seq_len=N, alpha=alpha, q=q, k=k, v=v, dout=dout, seq_offsets=off,
            num_targets=nt if targets else None, max_attn_len=max_attn_len, contextual_seq_len=ctx,
            min_full_attn_seq_len=min_full, ref_f32=res["f32"], ref_native=res["native"],
        ),
        os.path.join(HERE, f"attn_{name}.pt"),
    )


def delta_case(name, seed, B, H, max_uih, delta, dqk, dv, ctx, max_attn_len):
    g = torch.Generator().manual_seed(seed)
    lengths = torch.randint(1, max_uih + 1, (B,), generator=g) + delta + ctx
    N = max_uih + delta + ctx
    off = offsets_from(lengths.tolist())
    L = int(off[-1])
    nt = torch.full((B,), delta, dtype=torch.int64)
    k = torch.empty(L, H, dqk).uniform_(-0.1, 0.1, generator=g)
    v = torch.empty(L, H, dv).uniform_(-0.1, 0.1, generator=g)
    dq = torch.empty(B * delta, H, dqk).uniform_(-0.1, 0.1, generator=g)
    alpha = 1.0 / dqk**0.5
    out = delta_hstu_mha(max_seq_len=N, alpha=alpha, delta_q=dq, k=k, v=v, seq_offsets=off, num_targets=nt,
                         max_attn_len=max_attn_len, contextual_seq_len=ctx, kernel=PT)
    torch.save(dict(name=name, max_seq_len=N, alpha=alpha, delta_q=dq, k=k, v=v, seq_offsets=off, num_targets=nt,
                    max_attn_len=max_attn_len, contextual_seq_len=ctx, out=out),
               os.path.join(HERE, f"delta_{name}.pt"))


def ln_case(seed, N, D):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, D, generator=g)
    w = torch.randn(D, generator=g) * 0.5 + 1.0
    b = torch.randn(D, generator=g) * 0.1
    dy = torch.randn(N, D, generator=g)
    res = {}
    for nm, fn in (("ln", layer_norm), ("swish", swish_layer_norm)):
        xx, ww, bb = x.clone().requires_grad_(), w.clone().requires_grad_(), b.clone().requires_grad_()
        y = fn(xx, ww, bb, eps=1e-6, kernel=PT)
        y.backward(dy)
        res[nm] = dict(y=y.detach(), dx=xx.grad, dw=ww.grad, db=bb.grad)
    torch.save(dict(x=x, w=w, b=b, dy=dy, eps=1e-6, **res), os.path.join(HERE, f"layer_norm_{N}x{D}.pt"))


def output_case(name, seed, L, H, dv, D, group_norm, concat_ux):
    g = torch.Generator().manual_seed(seed)
    attn = torch.randn(L, H * dv, generator=g) * 0.3
    u = torch.randn(L, H * dv, generator=g)
    x = torch.randn(L, D, generator=g)
    nshape = H if group_norm else H * dv
    nw = torch.randn(nshape, generator=g) * 0.3 + 1.0
    nb = torch.randn(nshape, generator=g) * 0.1
    ow = torch.randn(H * dv * (3 if concat_ux else 1), D, generator=g) * 0.05
    dout = torch.randn(L, D, generator=g)
    ts = [t.clone().requires_grad_() for t in (attn, u, x, nw, nb, ow)]
    out = hstu_compute_output(
        attn=ts[0], u=ts[1], x=ts[2], norm_weight=ts[3], norm_bias=ts[4], norm_eps=1e-6, output_weight=ts[5],
        num_heads=H, linear_dim=dv, dropout_ratio=0.0, training=True, concat_ux=concat_ux, group_norm=group_norm,
        recompute_y_in_backward=False, kernel=PT,
    )
    out.backward(dout)
    torch.save(
        dict(name=name, attn=attn, u=u, x=x, norm_weight=nw, norm_bias=nb, output_weight=ow, dout=dout, eps=1e-6,
             num_heads=H, linear_dim=dv, group_norm=group_norm, concat_ux=concat_ux, out=out.detach(),
             grads=[t.grad for t in ts]),
        os.path.join(HERE, f"compute_output_{name}.pt"),
    )


def stu_case(name, seed, B, D, H, dqk, dv, layers, max_uih, max_tgt, group_norm, ctx, max_attn_len):
    torch.manual_seed(seed)
    random.seed(seed)
    stack = STUStack(
        [
            STULayer(
                STULayerConfig(embedding_dim=D, num_heads=H, hidden_dim=dv, attention_dim=dqk,
                               output_dropout_ratio=0.0, causal=True, target_aware=True,
                               max_attn_len=max_attn_len or None, attn_alpha=None, use_group_norm=group_norm,
                               recompute_normed_x=False, recompute_uvqk=False, recompute_y=False,
                               sort_by_length=False, contextual_seq_len=ctx)
            )
            for _ in range(layers)
        ]
    )
    stack.set_hammer_kernel(PT)
    # perturb the norm affine params so that their gradients are exercised
    with torch.no_grad():
        for n_, p in stack.named_parameters():
            if "norm_weight" in n_:
                p.add_(0.1 * torch.randn_like(p))
            if "norm_bias" in n_ or "beta" in n_:
                p.add_(0.05 * torch.randn_like(p))
    lengths = torch.randint(max_uih + 1, (B,))
    nt = torch.randint(1, max_tgt + 1, (B,))
    lengths = lengths + nt + ctx
    N = max_uih + max_tgt + ctx
    off = offsets_from(lengths.tolist())
    L = int(off[-1])
    x = torch.randn(L, D).requires_grad_()
    dout = torch.randn(L, D) * 0.1
    y = stack(x=x, x_lengths=lengths, x_offsets=off, max_seq_len=N, num_targets=nt)
    y.backward(dout)
    torch.save(
        dict(name=name, cfg=dict(embedding_dim=D, num_heads=H, hidden_dim=dv, attention_dim=dqk, layers=layers,
                                 use_group_norm=group_norm, contextual_seq_len=ctx, max_attn_len=max_attn_len),
             state_dict={k_: v_.detach().clone() for k_, v_ in stack.state_dict().items()},
             x=x.detach(), x_lengths=lengths, x_offsets=off, max_seq_len=N, num_targets=nt, dout=dout,
             y=y.detach(), dx=x.grad, param_grads={n_: p.grad for n_, p in stack.named_parameters()}),
        os.path.join(HERE, f"stu_{name}.pt"),
    )


def jagged_case(seed, B, D, max_l, max_r, ctx):
    g = torch.Generator().manual_seed(seed)
    ll = torch.randint(0, max_l + 1, (B,), generator=g)
    lr = torch.randint(ctx, max_r + 1, (B,), generator=g)
    ol, orr = offsets_from(ll.tolist()), offsets_from(lr.tolist())
    vl = torch.randn(int(ol[-1]), D, generator=g)
    vr = torch.randn(int(orr[-1]), D, generator=g)
    dense_r = torch.randn(B * max_r, D, generator=g)
    cat_jj = concat_2D_jagged(max_l + max_r, vl, vr, max_l, max_r, ol, orr, kernel=PT)
    cat_jd = concat_2D_jagged(max_l + max_r, vl, dense_r, max_l, max_r, ol, None, kernel=PT)
    sp_l, sp_r = split_2D_jagged(max_l + max_r, cat_jj, None, None, max_l, max_r, ol, orr, kernel=PT)
    sp_dl, sp_dr = split_2D_jagged(max_l + max_r, cat_jd, None, None, max_l, max_r, ol, None, kernel=PT)
    l2cat = hstu_concat_l2_embeddings(max_l, vl, ol, max_r, vr, orr, ctx, kernel=PT)
    l2_pre, l2_l2 = hstu_split_l2_embeddings(max_l + max_r, l2cat, ol, orr, ctx, kernel=PT)
    torch.save(dict(ol=ol, orr=orr, vl=vl, vr=vr, dense_r=dense_r, max_l=max_l, max_r=max_r, ctx=ctx,
                    cat_jj=cat_jj, cat_jd=cat_jd, sp_l=sp_l, sp_r=sp_r, sp_dl=sp_dl, sp_dr=sp_dr, l2cat=l2cat,
                    l2_pre=l2_pre, l2_l2=l2_l2), os.path.join(HERE, "jagged.pt"))


def research_case(seed, B, H, n, dqk, dv):
    from generative_recommenders.research.modeling.sequential.hstu import (
        RelativeBucketedTimeAndPositionBasedBias,
        _hstu_attention_maybe_from_cache,
    )

    torch.manual_seed(seed)
    lengths = torch.randint(1, n + 1, (B,))
    off = offsets_from(lengths.tolist())
    L = int(off[-1])
    q = torch.empty(L, H * dqk).uniform_(-0.3, 0.3).requires_grad_()
    k = torch.empty(L, H * dqk).uniform_(-0.3, 0.3).requires_grad_()
    v = torch.empty(L, H * dv).uniform_(-0.3, 0.3).requires_grad_()
    ts = torch.cumsum(torch.randint(0, 5000, (B, n)), dim=1)
    mod = RelativeBucketedTimeAndPositionBasedBias(
        max_seq_len=n, num_buckets=128,
        bucketization_fn=lambda x: (torch.log(torch.abs(x).clamp(min=1)) / 0.301).long(),
    )
    with torch.no_grad():
        mod._ts_w.normal_(0, 0.02)
        mod._pos_w.normal_(0, 0.02)
    mask = torch.triu(torch.ones(n, n, dtype=torch.bool), diagonal=1)
    invalid = 1.0 - mask.float()
    out, _, _ = _hstu_attention_maybe_from_cache(
        num_heads=H, attention_dim=dqk, linear_dim=dv, q=q, k=k, v=v, cached_q=None, cached_k=None,
        delta_x_offsets=None, x_offsets=off, all_timestamps=ts, invalid_attn_mask=invalid,
        rel_attn_bias=mod,
    )
    dout = torch.randn_like(out)
    out.backward(dout)
    torch.save(dict(n=n, H=H, dqk=dqk, dv=dv, q=q.detach(), k=k.detach(), v=v.detach(), seq_offsets=off,
                    timestamps=ts, pos_w=mod._pos_w.detach().clone(), ts_w=mod._ts_w.detach().clone(), dout=dout,
                    out=out.detach(), dq=q.grad, dk=k.grad, dv_=v.grad, dpos_w=mod._pos_w.grad,
                    dts_w=mod._ts_w.grad), os.path.join(HERE, "research_attn.pt"))


def research_block_case(name, seed, B, D, H, n, dqk, dv, concat_ua):
    """research/modeling/sequential/hstu.py:226-444 (SequentialTransductionUnitJagged.forward, no cache, eval-free: dropout 0)."""
    from generative_recommenders.research.modeling.sequential.hstu import (
        RelativeBucketedTimeAndPositionBasedBias,
        SequentialTransductionUnitJagged,
    )

    torch.manual_seed(seed)
    lengths = torch.randint(1, n + 1, (B,))
    off = offsets_from(lengths.tolist())
    L = int(off[-1])
    x = torch.randn(L, D).requires_grad_()
    ts = torch.cumsum(torch.randint(0, 5000, (B, n)), dim=1)
    bias_mod = RelativeBucketedTimeAndPositionBasedBias(
        max_seq_len=n, num_buckets=128,
        bucketization_fn=lambda t: (torch.log(torch.abs(t).clamp(min=1)) / 0.301).long(),
    )
    with torch.no_grad():
        bias_mod._ts_w.normal_(0, 0.02)
        bias_mod._pos_w.normal_(0, 0.02)
    blk = SequentialTransductionUnitJagged(
        embedding_dim=D, linear_hidden_dim=dv, attention_dim=dqk, dropout_ratio=0.0, attn_dropout_ratio=0.0, num_heads=H,
        linear_activation="silu", relative_attention_bias_module=bias_mod, normalization="rel_bias", linear_config="uvqk",
        concat_ua=concat_ua, epsilon=1e-6, max_length=n,
    )
    with torch.no_grad():
        blk._uvqk.normal_(0, 0.1)
        blk._o.bias.normal_(0, 0.1)
    invalid = torch.tril(torch.ones(n, n))
    y, _ = blk(x, off, ts, invalid)
    dy = torch.randn_like(y)
    y.backward(dy)
    torch.save(dict(n=n, H=H, D=D, dqk=dqk, dv=dv, concat_ua=concat_ua, eps=1e-6, x=x.detach(), seq_offsets=off, timestamps=ts,
                    state_dict={k: v.detach().clone() for k, v in blk.state_dict().items()}, dy=dy, y=y.detach(), dx=x.grad,
                    grads={k: p_.grad.detach().clone() for k, p_ in blk.named_parameters()}),
               os.path.join(HERE, f"research_block_{name}.pt"))


def position_case(name, seed, B, max_uih, max_targets, D, max_ctx, interleave, bucket_fn, dtype, with_targets=True):
    # input recipe of ops/tests/position_test.py:96-170; eager path ops/position.py:43-96 -> ops/pytorch/pt_position.py:75-134
    from generative_recommenders.ops.position import add_timestamp_positional_embeddings

    g = torch.Generator().manual_seed(seed)
    alpha = 0.5 if seed % 2 else 1.7
    num_targets = torch.randint(max_targets + 1, (B,), generator=g)
    lengths = torch.randint(max_uih + 1, (B,), generator=g) + num_targets * (2 if interleave else 1)
    lengths[0] = max(int(lengths[0]), 1)
    off = offsets_from(lengths.tolist())
    max_seq_len = max_uih + max_targets * (2 if interleave else 1)
    pos_w = torch.empty(max_seq_len, D).uniform_(-1.0, 1.0, generator=g).requires_grad_()
    ts_w = torch.empty(200, D).uniform_(-1.0, 1.0, generator=g).requires_grad_()  # the reference test uses 1000 rows; 200 > D - 1 keeps the fixture small
    x = torch.empty(int(off[-1]), D).uniform_(-0.1, 0.1, generator=g).to(dtype).requires_grad_()
    deltas = torch.randint(86400, (B, max_seq_len), generator=g)
    ts_dense = deltas.cumsum(dim=1)
    mask = torch.arange(max_seq_len) < lengths.unsqueeze(1)
    ts = ts_dense[mask]
    out = add_timestamp_positional_embeddings(
        alpha=alpha, max_seq_len=max_seq_len, max_contextual_seq_len=max_ctx, position_embeddings_weight=pos_w,
        timestamp_embeddings_weight=ts_w, seq_offsets=off, seq_lengths=lengths, seq_embeddings=x, timestamps=ts,
        num_targets=num_targets if with_targets else None, interleave_targets=interleave, time_bucket_fn=bucket_fn, kernel=PT)
    dout = (torch.randn(out.shape, generator=g) * 0.01).to(out.dtype)
    out.backward(dout)
    torch.save(dict(name=name, alpha=alpha, max_seq_len=max_seq_len, max_contextual_seq_len=max_ctx, interleave_targets=interleave,
                    time_bucket_fn=bucket_fn, pos_w=pos_w.detach(), ts_w=ts_w.detach(), seq_offsets=off, seq_lengths=lengths,
                    x=x.detach(), timestamps=ts, num_targets=num_targets if with_targets else None, dout=dout, out=out.detach(),
                    dx=x.grad, dpos_w=pos_w.grad, dts_w=ts_w.grad),
               os.path.join(HERE, f"position_{name}.pt"))


def ssl_case(name, seed, B, N, D, R, V, l2_norm, temperature, dtype):
    # research/modeling/sequential/losses/sampled_softmax.py:91-193 (dense forward -> jagged_forward) with the sampler and the
    # similarity the HSTU configs use (LocalNegativesSampler, DotProductSimilarity)
    from generative_recommenders.research.modeling.sequential.autoregressive_losses import LocalNegativesSampler
    from generative_recommenders.research.modeling.sequential.losses.sampled_softmax import SampledSoftmaxLoss
    from generative_recommenders.research.rails.similarities.dot_product_similarity_fn import DotProductSimilarity

    class _Model(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self._sim = DotProductSimilarity()

        def similarity_fn(self, query_embeddings, item_ids, item_embeddings, **kwargs):
            return self._sim(query_embeddings=query_embeddings, item_embeddings=item_embeddings)

    torch.manual_seed(seed)
    emb = torch.nn.Embedding(V, D)
    with torch.no_grad():
        emb.weight.normal_(0, 0.3)
        emb.weight[3].mul_(1e-9)  # one row whose norm is clamped by l2_norm_eps
    emb = emb.to(dtype)
    sampler = LocalNegativesSampler(num_items=V, item_emb=emb, all_item_ids=list(range(V)), l2_norm=l2_norm, l2_norm_eps=1e-6)
    loss_mod = SampledSoftmaxLoss(num_to_sample=R, softmax_temperature=temperature, model=_Model())
    lengths = torch.randint(1, N + 1, (B,))
    out = (torch.randn(B, N, D) * 0.5).to(dtype).requires_grad_()
    ids = torch.randint(0, V, (B, N))
    ids[0, 0] = 3
    sup = emb(ids).detach().clone().requires_grad_()
    w = (torch.rand(B, N) > 0.2).float() * torch.rand(B, N)
    gen_state = torch.get_rng_state()
    loss, _ = loss_mod(lengths=lengths, output_embeddings=out, supervision_ids=ids, supervision_embeddings=sup,
                       supervision_weights=w.to(dtype), negatives_sampler=sampler)
    loss.backward()
    # the ids the sampler drew (same generator state, same call)
    torch.set_rng_state(gen_state)
    keep = torch.arange(N).unsqueeze(0) < lengths.unsqueeze(1)
    sampled = torch.randint(low=0, high=V, size=(int(keep.sum()), R), dtype=ids.dtype)
    torch.save(dict(name=name, R=R, V=V, l2_norm=l2_norm, l2_norm_eps=1e-6, temperature=temperature, lengths=lengths,
                    output_embeddings=out.detach(), supervision_ids=ids, supervision_embeddings=sup.detach(), weights=w.to(dtype),
                    table=emb.weight.detach().clone(), rng_state=gen_state, sampled_ids=sampled, loss=loss.detach(),
                    d_out=out.grad, d_sup=sup.grad, d_table=emb.weight.grad),
               os.path.join(HERE, f"ssl_{name}.pt"))


def jagged_bmm_case(name, seed, B, max_len, K, N, dtype):
    # ops/tests/jagged_tensors_test.py:_test_jagged_dense_bmm_broadcast_add recipe; eager path ops/pytorch/pt_jagged.py:77-98
    from generative_recommenders.ops.jagged_tensors import jagged_dense_bmm_broadcast_add

    g = torch.Generator().manual_seed(seed)
    lengths = torch.randint(max_len + 1, (B,), generator=g)
    lengths[0] = 0
    off = offsets_from(lengths.tolist())
    L = int(off[-1])
    jag = torch.empty(L, K).uniform_(-1, 1, generator=g).to(dtype).requires_grad_()
    dense = torch.empty(B, K, N).uniform_(-1, 1, generator=g).to(dtype).requires_grad_()
    bias = torch.empty(B, N).uniform_(-1, 1, generator=g).to(dtype).requires_grad_()
    out = jagged_dense_bmm_broadcast_add(max_seq_len=max_len, seq_offsets=off, jagged=jag, dense=dense, bias=bias, kernel=PT)
    dout = torch.randn(out.shape, generator=g).to(dtype) * 0.1
    out.backward(dout)
    torch.save(dict(name=name, max_seq_len=max_len, seq_offsets=off, jagged=jag.detach(), dense=dense.detach(), bias=bias.detach(),
                    dout=dout, out=out.detach(), d_jagged=jag.grad, d_dense=dense.grad, d_bias=bias.grad),
               os.path.join(HERE, f"jagged_bmm_{name}.pt"))


def research_cache_case(seed, B, D, H, n, dqk, dv):
    # research/modeling/sequential/hstu.py:284-444 with delta_x_offsets / cache: full forward with return_cache_states=True,
    # then the LAST row of every sequence is replaced and only those rows are recomputed against the cache
    from generative_recommenders.research.modeling.sequential.hstu import (
        RelativeBucketedTimeAndPositionBasedBias,
        SequentialTransductionUnitJagged,
    )

    torch.manual_seed(seed)
    lengths = torch.randint(2, n + 1, (B,))
    off = offsets_from(lengths.tolist())
    L = int(off[-1])
    x = torch.randn(L, D)
    ts = torch.cumsum(torch.randint(0, 5000, (B, n)), dim=1)
    bias_mod = RelativeBucketedTimeAndPositionBasedBias(
        max_seq_len=n, num_buckets=128, bucketization_fn=lambda t: (torch.log(torch.abs(t).clamp(min=1)) / 0.301).long())
    with torch.no_grad():
        bias_mod._ts_w.normal_(0, 0.02)
        bias_mod._pos_w.normal_(0, 0.02)
    blk = SequentialTransductionUnitJagged(
        embedding_dim=D, linear_hidden_dim=dv, attention_dim=dqk, dropout_ratio=0.0, attn_dropout_ratio=0.0, num_heads=H,
        linear_activation="silu", relative_attention_bias_module=bias_mod, normalization="rel_bias", linear_config="uvqk",
        concat_ua=False, epsilon=1e-6, max_length=n)
    with torch.no_grad():
        blk._uvqk.normal_(0, 0.1)
        blk._o.bias.normal_(0, 0.1)
    blk.eval()
    invalid = torch.tril(torch.ones(n, n))
    with torch.no_grad():
        y0, cache = blk(x, off, ts, invalid, return_cache_states=True)
        x2 = x.clone()
        last_rows = off[1:] - 1
        x2[last_rows] = torch.randn(B, D)
        delta = (last_rows.clone(), (lengths - 1).clone())
        cache_in = tuple(t.clone() for t in cache)
        y1, cache1 = blk(x2, off, ts, invalid, delta_x_offsets=delta, cache=tuple(t.clone() for t in cache))
        y_full, _ = blk(x2, off, ts, invalid)  # what a full forward on the updated input gives (rows other than the last differ only
        #                                        through the cache semantics: they keep their cached outputs)
    torch.save(dict(n=n, H=H, D=D, dqk=dqk, dv=dv, x=x, x2=x2, seq_offsets=off, timestamps=ts, delta_rows=delta[0], delta_pos=delta[1],
                    state_dict={k: v.detach().clone() for k, v in blk.state_dict().items()}, y0=y0, cache0=cache_in, y1=y1,
                    cache1=tuple(t.clone() for t in cache1), y_full=y_full),
               os.path.join(HERE, "research_block_cache.pt"))


def main():
    only = set(sys.argv[1:])
    if not only or "research_cache" in only:
        research_cache_case(75, 3, 32, 2, 24, 16, 16)
    if not only or "jagged_bmm" in only:
        jagged_bmm_case("f32", 95, 5, 40, 24, 36, torch.float32)
        jagged_bmm_case("bf16", 96, 4, 70, 64, 80, torch.bfloat16)
    if not only or "ssl" in only:
        ssl_case("l2_f32", 91, 4, 12, 64, 16, 50, True, 0.05, torch.float32)
        ssl_case("plain_f32", 92, 3, 9, 32, 8, 40, False, 1.0, torch.float32)
        ssl_case("l2_bf16", 93, 4, 10, 64, 32, 64, True, 0.05, torch.bfloat16)  # e.g. `make_golden.py position`: regenerate only the named groups
    if not only or "position" in only:
        position_case("log_f32", 81, 5, 60, 10, 40, 0, False, "log", torch.float32)
        position_case("sqrt_ctx_bf16", 82, 6, 90, 8, 64, 5, False, "sqrt", torch.bfloat16)
        position_case("log_interleave_f16", 83, 4, 50, 6, 24, 3, True, "log", torch.float16)
        position_case("sqrt_d136", 84, 4, 70, 5, 136, 0, False, "sqrt", torch.float32)
    if only:
        print("golden vectors written to", HERE, "for", sorted(only))
        return
    f32, bf16 = torch.float32, torch.bfloat16
    #          name        seed B  H  uih tgt dqk dv  targets  mal ctx min_full dtype
    attn_case("plain", 1, 4, 2, 40, 6, 16, 16, False, 0, 0, 0, f32)
    attn_case("targets", 2, 5, 3, 70, 9, 32, 16, True, 0, 0, 0, f32)
    attn_case("window", 3, 4, 2, 90, 7, 16, 32, True, 11, 0, 0, f32)
    attn_case("context", 4, 4, 2, 60, 5, 24, 24, True, 0, 6, 0, f32)
    attn_case("ctx_window_full", 5, 4, 1, 100, 8, 16, 16, True, 9, 4, 13, f32)
    attn_case("bf16_d64", 6, 3, 2, 150, 10, 64, 64, True, 0, 0, 0, bf16)
    attn_case("bf16_d32_window", 7, 3, 4, 200, 12, 32, 32, True, 25, 3, 0, bf16)
    attn_case("odd_dims", 8, 3, 2, 33, 4, 25, 50, True, 0, 0, 0, f32)
    delta_case("plain", 11, 4, 2, 50, 7, 16, 32, 0, 0)
    delta_case("ctx", 12, 3, 2, 40, 5, 32, 16, 4, 0)
    ln_case(21, 37, 64)
    ln_case(22, 50, 200)
    output_case("ln_concat", 31, 45, 2, 16, 24, False, True)
    output_case("gn_concat", 32, 45, 4, 8, 24, True, True)
    output_case("ln_plain", 33, 30, 2, 16, 24, False, False)
    stu_case("ln", 41, 4, 32, 2, 16, 16, 2, 30, 5, False, 0, 0)
    stu_case("gn_ctx_window", 42, 4, 48, 4, 8, 16, 2, 40, 6, True, 3, 9)
    jagged_case(51, 6, 8, 9, 12, 2)
    research_case(61, 3, 2, 24, 16, 16)
    research_block_case("plain", 71, 3, 32, 2, 24, 16, 16, False)
    research_block_case("concat_ua", 72, 4, 48, 4, 20, 8, 16, True)
    print("golden vectors written to", HERE)


if __name__ == "__main__":
    main()
