"""Torch emulation of the FP8 encoder path (bert_precision='fp8'): the same quantisation as the kernels, with block scales
and per-block promotion in float64.

  scale = amax / 448 in fp32 (1 when amax == 0);  q = clamp(x / scale, -448, 448) -> float8_e4m3fn (round to nearest even).
The clamp is required: torch's cast turns values above 464 into NaN, the kernels saturate at 448.
  weights      per output channel: s_w[n] = max_k |W[k,n]| / 448, q [N,K]
  activations  per 1 x 128 block:  s_a[m,j] over row m, columns [128j, 128j+128), q [M,K]
  GEMM         s_w[n] * sum_j s_a[m,j] * (qa_j . qw_j) + bias[n]

The encoder is oracle/nn.py's bert_encoder with the QKV, FFN1 and FFN2 GEMMs replaced by that emulation, and bf16 rounding
where the bf16 path rounds (qkv, the attention context and probabilities, the out-projection and FFN2 outputs).  Works on
any device; float64 throughout apart from the fp32 scale / quantisation steps the kernels perform in fp32.
"""
import math

import torch

from oracle import nn as onn

E4M3 = torch.float8_e4m3fn
E4M3_MAX = 448.0


def scale_of(amax):
    amax = amax.to(torch.float32)
    # tensor / tensor: torch divides by a Python scalar as a multiplication by its reciprocal, which is not the correctly
    # rounded amax / 448 the kernels compute
    return torch.where(amax > 0, amax / torch.full_like(amax, E4M3_MAX), torch.ones_like(amax))


def quant(x, s):
    return torch.clamp(x.to(torch.float32) / s, -E4M3_MAX, E4M3_MAX).to(E4M3)


def quantize_weight(w_kn):
    """TF kernel [K,N] -> (e4m3 [N,K], f32 scales [N])."""
    w = w_kn.to(torch.float32)
    s = scale_of(w.abs().amax(0))
    return quant(w, s[None, :]).t().contiguous(), s


def quantize_rows(x):
    """[M,K] (quantised from its fp32 value) -> (e4m3 [M,K], f32 block scales [M, K/128])."""
    M, K = x.shape
    xb = x.to(torch.float32).reshape(M, K // 128, 128)
    s = scale_of(xb.abs().amax(-1))
    return quant(xb, s[..., None]).reshape(M, K), s


def dequant_gemm(qa, sa, qw, sw, bias=None):
    """float64 s_w[n] * sum_j s_a[m,j] * (qa_j . qw_j) (+ bias): each product qa * s_a is exact in float64."""
    M, K = qa.shape
    a = (qa.to(torch.float64).reshape(M, K // 128, 128) * sa.to(torch.float64)[..., None]).reshape(M, K)
    y = (a @ qw.to(torch.float64).t()) * sw.to(torch.float64)
    return y if bias is None else y + bias.to(torch.float64)


def gelu_e4m3(y, variant):
    """GELU of a float64 pre-activation, quantised per 1 x 128 block -> (e4m3, scales)."""
    return quantize_rows(onn.gelu(y, variant))


def bert_encoder_fp8(w, input_ids, input_mask, segment_ids, num_layers, num_heads=12, gelu_variant="tanh", prefix="bert",
                     device="cpu"):
    """sequence_output [B,L,H] float64 of the FP8 encoder."""
    g = lambda name: w[f"{prefix}/{name}"].to(device=device, dtype=torch.float64)
    rb = lambda t: onn._rb(t, True)
    ids = input_ids.long().to(device)
    B, L = ids.shape
    seg = torch.zeros_like(ids) if segment_ids is None else segment_ids.long().to(device)
    x = g("embeddings/word_embeddings")[ids] + g("embeddings/token_type_embeddings")[seg] \
        + g("embeddings/position_embeddings")[:L][None]
    x = onn.layer_norm(x, g("embeddings/LayerNorm/gamma"), g("embeddings/LayerNorm/beta"), 1e-12).reshape(B * L, -1)
    H = x.shape[-1]
    dh = H // num_heads
    adder = (1.0 - input_mask.to(device=device, dtype=torch.float64))[:, None, None, :] * -10000.0
    sh = lambda t: t.view(B, L, num_heads, dh).permute(0, 2, 1, 3)
    for l in range(num_layers):
        p = f"encoder/layer_{l}"
        wk = lambda name: w[f"{prefix}/{p}/{name}"].to(device=device, dtype=torch.float32)
        wqkv = torch.cat([wk(f"attention/self/{n}/kernel") for n in ("query", "key", "value")], dim=1)
        bqkv = torch.cat([wk(f"attention/self/{n}/bias") for n in ("query", "key", "value")])
        xq, xs = quantize_rows(x)
        qkv = rb(dequant_gemm(xq, xs, *quantize_weight(wqkv), bqkv))
        q, k, v = qkv[:, :H], qkv[:, H:2 * H], qkv[:, 2 * H:]
        scores = sh(q) @ sh(k).transpose(-1, -2) * (1.0 / math.sqrt(dh)) + adder
        m = scores.max(-1, keepdim=True).values
        e = torch.exp(scores - m)
        ctx = rb(((rb(e) @ sh(v)) / e.sum(-1, keepdim=True)).permute(0, 2, 1, 3).reshape(B * L, H))
        a = rb(onn.dense(ctx, rb(g(f"{p}/attention/output/dense/kernel")), g(f"{p}/attention/output/dense/bias")))
        x1 = onn.layer_norm(a + x, g(f"{p}/attention/output/LayerNorm/gamma"), g(f"{p}/attention/output/LayerNorm/beta"), 1e-12)
        x1q, x1s = quantize_rows(x1)
        hq, hs = gelu_e4m3(dequant_gemm(x1q, x1s, *quantize_weight(wk("intermediate/dense/kernel")), wk("intermediate/dense/bias")),
                           gelu_variant)
        o = rb(dequant_gemm(hq, hs, *quantize_weight(wk("output/dense/kernel")), wk("output/dense/bias")))
        x = onn.layer_norm(o + x1, g(f"{p}/output/LayerNorm/gamma"), g(f"{p}/output/LayerNorm/beta"), 1e-12)
    return x.view(B, L, H)
