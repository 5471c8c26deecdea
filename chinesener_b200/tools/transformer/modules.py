# -*-coding:utf-8 -*-
"""Transformer building blocks with the reference's surface (reference tools/transformer/modules.py),
executed at fp32 accuracy: dense layers run as three split-bf16 wgmma products (ops.gemm_split_f32),
LayerNorm / attention in fp32."""
import numpy as np
import torch

from ... import autodiff, ops, variables

FP32_EPS = float(np.finfo(np.float32).eps)


def _dense_pack(store, name, K, N):
    """(w_hi, w_lo) bf16 [N, K8] packs of the TF kernel `name/kernel` [K, N] (K zero-padded to a multiple of 8)."""
    Kp = (K + 7) // 8 * 8

    def build():
        w = store.vars[f"{name}/kernel"]
        if Kp != K:
            w = torch.nn.functional.pad(w, (0, 0, 0, Kp - K))
        w = w.contiguous()
        hi = ops.pack_weight_bf16(w)                                   # [N, Kp] bf16
        lo = ops.pack_weight_bf16((w - hi.float().t()).contiguous())
        return hi, lo, Kp
    return store.cached(("dense_split_pack", name, K, N), build)


def dense_f32(x2d, units, name, relu=False, residual=None, use_bias=True):
    """tf.layers.dense(x, units, name=name) on a [M, K] f32 activation at fp32 accuracy -> f32 [M, units]."""
    M, K = x2d.shape
    assert units % 32 == 0, "split-bf16 dense path needs units % 32 == 0"
    store = variables.default_store()
    store.get_variable(f"{name}/kernel", (K, units), variables.glorot_uniform)
    b = store.get_variable(f"{name}/bias", (units,), variables.zeros) if use_bias else None
    w_hi, w_lo, Kp = _dense_pack(store, name, K, units)
    a_hi, a_lo = ops.split_bf16(x2d, Kp)
    return ops.gemm_split_f32(a_hi, a_lo, w_hi, w_lo, b, residual=residual, relu=relu)


def dense_train(x2d, units, name, relu=False):
    """TRAIN-mode tf.layers.dense: same forward as dense_f32, records dW = x^T·dy, db = colsum(dy), dx = dy·W^T
    (tensor-core GEMMs on bf16 casts of the f32 gradients, fp32 accumulation)."""
    store, tape = variables.default_store(), autodiff.current()
    y = dense_f32(x2d, units, name, relu=relu)
    need_dx = tape.needs_grad(x2d)

    def bwd(g):
        if g is None:
            return
        g = g.contiguous()
        if relu:
            g = ops.relu_bwd(y, g)
        ops.colsum_add(g, store.grad(f"{name}/bias"))
        ops.wgrad_gemm(x2d, g, out=store.grad(f"{name}/kernel"))
        if need_dx:                                                  # W [K,N] in TF layout is the K-major operand of dy·W^T
            tape.add_grad(x2d, ops.gemm_bf16(ops.cast_bf16(g), ops.cast_bf16(store.vars[f"{name}/kernel"]), None,
                                             epilogue=ops.EPI_F32))
    tape.record(y, bwd)
    return y


def add_and_norm_train(x2d, y2d, scope, dropout_rate):
    """layer_norm(x + dropout(y)) (reference modules.py:23-37 after the sub-layer's tf.layers.dropout), dropout fused
    into the LayerNorm kernels; gradients: residual branch -> x, masked branch -> y."""
    store, tape = variables.default_store(), autodiff.current()
    d = x2d.shape[-1]
    kn, bn = f"{scope}/layer_normalization/norm_kernel", f"{scope}/layer_normalization/norm_bias"
    k = store.get_variable(kn, (d,), variables.ones)
    b = store.get_variable(bn, (d,), variables.zeros)
    keep = 1.0 - float(dropout_rate)
    store.dropout_calls += 1
    seed = (777 * 1000003 + store.global_step) * 1009 + store.dropout_calls
    out, _ = ops.layernorm(y2d, k, b, residual=x2d, eps=FP32_EPS, want_bf16=False, keep_prob=keep, seed=seed)

    def bwd(g):
        if g is None:
            return
        dz32, dz16 = ops.layernorm_bwd(y2d, k, g.contiguous(), store.grad(kn), store.grad(bn), residual=x2d, eps=FP32_EPS,
                                       want_bf16=keep < 1.0, keep_prob=keep, seed=seed)
        tape.add_grad(x2d, dz32)
        tape.add_grad(y2d, dz32 if keep >= 1.0 else dz16.float())
    tape.record(out, bwd)
    return out


def embedding_project(embedding2d, d_model, name='embedding/dense', is_training=False):
    """reference modules.py:11-20 — linear map of the raw char(+bichar) embedding to d_model."""
    if embedding2d.shape[-1] == d_model:
        return embedding2d
    if is_training:
        return dense_train(embedding2d, d_model, name)
    return dense_f32(embedding2d, d_model, name)


def layer_norm(x2d, scope):
    """reference modules.py:40-65 — (x-mean)/sqrt(var+eps)*norm_kernel+norm_bias, eps = fp32 machine eps."""
    d = x2d.shape[-1]
    k = variables.get_variable(f"{scope}/layer_normalization/norm_kernel", (d,), variables.ones)
    b = variables.get_variable(f"{scope}/layer_normalization/norm_bias", (d,), variables.zeros)
    out, _ = ops.layernorm(x2d, k, b, eps=FP32_EPS, want_bf16=False)
    return out


def ffn(x2d, ffn_hidden, dropout_rate, is_training, scope):
    """reference modules.py:68-80 — dense-relu-dense (+dropout when training) + add & norm."""
    d_model = x2d.shape[-1]
    if is_training:
        y = dense_train(x2d, ffn_hidden, f"{scope}/ffn/ffn_inner", relu=True)
        y = dense_train(y, d_model, f"{scope}/ffn/ffn_outer")
        return add_and_norm_train(x2d, y, f"{scope}/ffn/add_and_norm", dropout_rate)
    y = dense_f32(x2d, ffn_hidden, f"{scope}/ffn/ffn_inner", relu=True)
    y = dense_f32(y, d_model, f"{scope}/ffn/ffn_outer", residual=x2d)          # x + y fused into the epilogue
    return layer_norm(y, f"{scope}/ffn/add_and_norm")


def sinusoidal_positional_encoding(emb_dim, pos_seq):
    """reference modules.py:177-197 — numpy table, cast to float32 exactly like the reference."""
    inv_freq = np.array([1 / (10000 ** ((i - i % 2) / emb_dim)) for i in range(emb_dim)])
    enc = np.einsum('i,j->ij', np.asarray(pos_seq, dtype=np.float64), inv_freq)
    out = np.where(np.arange(emb_dim)[None, :] % 2 == 1, np.cos(enc), np.sin(enc))
    return out.astype(np.float32)


def multi_head_attention(x2d, seq_len, B, L, num_head, dropout_rate, is_training, scope):
    """reference modules.py:129-175 with key = value = query = x: projected K/V/Q, scaled dot product over the valid
    keys (fp32 attention kernel), output projection, dropout, add & norm."""
    d_model = x2d.shape[-1]
    dh = d_model // num_head
    p = f"{scope}/multi_head_attention"
    dense = dense_train if is_training else dense_f32
    k = dense(x2d, d_model, f"{p}/pre_key_project")
    v = dense(x2d, d_model, f"{p}/pre_value_project")
    q = dense(x2d, d_model, f"{p}/pre_query_project")
    scale = dh ** -0.5
    ctx, _, _ = ops.attention_f32(q, k, v, seq_len, B, L, num_head, dh, scale=scale)
    if not is_training:
        y = dense_f32(ctx, d_model, f"{p}/post_linear_project", residual=x2d)
        return layer_norm(y, f"{p}/add_and_norm")
    tape = autodiff.current()

    def bwd(g):
        if g is None:
            return
        dq, dk, dv, _, _ = ops.attention_f32_bwd(q, k, v, seq_len, B, L, num_head, dh, g.contiguous(), scale=scale)
        tape.add_grad(q, dq)
        tape.add_grad(k, dk)
        tape.add_grad(v, dv)
    tape.record(ctx, bwd)
    y = dense_train(ctx, d_model, f"{p}/post_linear_project")
    return add_and_norm_train(x2d, y, f"{p}/add_and_norm", dropout_rate)
