"""The FP8 entry points (ner_gemm_e4m3, ner_quantize_weight_e4m3, the e4m3 LayerNorms, ner_bert_encoder_fwd_fp8) are
registered and reject bad arguments before any CUDA call, so this runs without a GPU."""
import ctypes

from chinesener_b200 import _lib

FP8_ENTRIES = ("ner_gemm_e4m3", "ner_quantize_weight_e4m3", "ner_bert_embed_ln_e4m3", "ner_layernorm_e4m3",
               "ner_bert_encoder_fp8_workspace_bytes", "ner_bert_encoder_fwd_fp8")
EPI_BF16, EPI_GELU_TANH_E4M3, EPI_GELU_ERF_E4M3 = 1, 7, 8


def test_fp8_signatures_registered():
    h = _lib.lib()
    for name in FP8_ENTRIES:
        assert name in _lib.SIGNATURES
        assert getattr(h, name).argtypes == _lib.SIGNATURES[name][1]


def test_gemm_e4m3_argument_checks():
    f = _lib.lib().ner_gemm_e4m3
    # (A, a_scale, Wt, w_scale, bias, out, out_scale, M, N, K, epilogue, stream); 4096 = a 16-byte aligned fake pointer
    p = 4096
    assert f(p, p, p, p, p, p, p, -1, 128, 128, EPI_BF16, None) == -1         # negative M
    assert f(p, p, p, p, p, p, p, 8, 0, 128, EPI_BF16, None) == -1            # N = 0
    assert f(p, p, p, p, p, p, p, 8, 128, 0, EPI_BF16, None) == -1            # K = 0
    assert f(p, p, p, p, p, p, p, 8, 128, 128, 0, None) == -1                 # f32 epilogue: not an FP8 mode
    assert f(p, p, p, p, p, p, p, 8, 128, 128, 2, None) == -1                 # bf16 GELU epilogue: not an FP8 mode
    assert f(p, p, p, p, p, p, p, 8, 128, 100, EPI_BF16, None) == -2          # K % 128 != 0
    assert f(p, p, p, p, p, p, p, 8, 128, 192, EPI_BF16, None) == -2          # K % 128 != 0
    assert f(p, p, p, p, p, p, p, 8, 96, 128, EPI_BF16, None) == -2           # N % 128 != 0
    assert f(None, None, None, None, None, None, None, 0, 128, 128, EPI_BF16, None) == 0   # M = 0: no-op
    assert f(None, p, p, p, p, p, p, 8, 128, 128, EPI_BF16, None) == -1       # null A
    assert f(p, None, p, p, p, p, p, 8, 128, 128, EPI_BF16, None) == -1       # null a_scale
    assert f(p, p, None, p, p, p, p, 8, 128, 128, EPI_BF16, None) == -1       # null Wt
    assert f(p, p, p, None, p, p, p, 8, 128, 128, EPI_BF16, None) == -1       # null w_scale
    assert f(p, p, p, p, p, None, p, 8, 128, 128, EPI_BF16, None) == -1       # null out
    for epi in (EPI_GELU_TANH_E4M3, EPI_GELU_ERF_E4M3):
        assert f(p, p, p, p, p, p, None, 8, 128, 128, epi, None) == -1        # e4m3 output needs out_scale
    assert f(p + 8, p, p, p, p, p, p, 8, 128, 128, EPI_BF16, None) == -1      # A not 16-byte aligned
    assert f(p, p, p, p + 4, p, p, p, 8, 128, 128, EPI_BF16, None) == -1      # w_scale not 8-byte aligned
    assert f(p, p, p, p, p + 4, p, p, 8, 128, 128, EPI_BF16, None) == -1      # bias not 8-byte aligned


def test_quantize_weight_argument_checks():
    f = _lib.lib().ner_quantize_weight_e4m3
    # (w_kn, wt_nk_e4m3, w_scale, K, N, stream)
    assert f(1, 1, 1, 0, 8, None) == -1
    assert f(1, 1, 1, 8, 0, None) == -1
    assert f(None, 1, 1, 8, 8, None) == -1
    assert f(1, None, 1, 8, 8, None) == -1
    assert f(1, 1, None, 8, 8, None) == -1


def test_layernorm_e4m3_argument_checks():
    f = _lib.lib().ner_layernorm_e4m3
    # (y, y_is_bf16, residual, gamma, beta, out_f32, out_bf16, out_e4m3, out_scale, M, H, eps, stream)
    assert f(1, 1, None, 1, 1, 1, None, 1, 1, -1, 768, 1e-12, None) == -1     # negative M
    assert f(None, 1, None, None, None, None, None, None, None, 0, 768, 1e-12, None) == 0   # M = 0: no-op
    assert f(1, 1, None, 1, 1, 1, None, None, 1, 4, 768, 1e-12, None) == -1   # null e4m3 output
    assert f(1, 1, None, 1, 1, 1, None, 1, None, 4, 768, 1e-12, None) == -1   # null scale output
    assert f(None, 1, None, 1, 1, 1, None, 1, 1, 4, 768, 1e-12, None) == -1   # null y
    assert f(1, 1, None, 1, 1, 1, None, 1, 1, 4, 320, 1e-12, None) == -2      # H % 128 != 0
    assert f(1, 1, None, 1, 1, 1, None, 1, 1, 4, 1152, 1e-12, None) == -2     # H > 1024
    g = _lib.lib().ner_bert_embed_ln_e4m3
    # (word, type, pos, gamma, beta, ids, seg, out_f32, out_bf16, out_e4m3, out_scale, B, L, H, vocab, n_type, max_pos, eps,
    #  tok_src, n_packed, stream)
    assert g(1, 1, 1, 1, 1, 1, None, 1, None, None, 1, 2, 8, 768, 100, 2, 512, 1e-12, None, 0, None) == -1   # null e4m3 out
    assert g(1, 1, 1, 1, 1, 1, None, 1, None, 1, None, 2, 8, 768, 100, 2, 512, 1e-12, None, 0, None) == -1   # null scales
    assert g(1, 1, 1, 1, 1, 1, None, 1, None, 1, 1, 2, 8, 320, 100, 2, 512, 1e-12, None, 0, None) == -2     # H % 128 != 0
    assert g(1, 1, 1, 1, 1, 1, None, 1, None, 1, 1, -1, 8, 768, 100, 2, 512, 1e-12, None, 0, None) == -1    # negative B


def _cfg(H=768, I=3072, NH=12, layers=12):
    return _lib.BertConfig(H, NH, I, layers, 21128, 2, 512, 1e-12, 0, 0)


def test_encoder_fp8_argument_checks():
    h = _lib.lib()
    ws = h.ner_bert_encoder_fp8_workspace_bytes
    assert ws(ctypes.byref(_cfg()), 0) == 0
    assert ws(ctypes.byref(_cfg()), 4096) > ws(ctypes.byref(_cfg()), 1024) > 0
    assert ws(None, 8) == 0 and ws(ctypes.byref(_cfg()), -1) == 0
    f = h.ner_bert_encoder_fwd_fp8
    layers = (_lib.BertLayerWeightsFp8 * 12)()

    def call(cfg, B=2, L=8, out=1, lay=layers, ws_bytes=1 << 30, cu=None, tok=None, n=0):
        return f(ctypes.byref(cfg), 1, 1, 1, 1, 1, lay, 1, 1, None, B, L, cu, tok, n, out, out, 1, ws_bytes, None)
    assert call(_cfg(H=704, NH=11)) == -2                # hidden_size % 128 != 0
    assert call(_cfg(I=3000)) == -2                      # intermediate_size % 128 != 0
    assert call(_cfg(), out=None) == -1                  # null outputs
    assert call(_cfg(), lay=None) == -1                  # null layer table
    assert call(_cfg(), B=-1) == -1
    assert call(_cfg(), L=0) == -1
    assert call(_cfg(H=768, NH=7)) == -1                 # heads do not divide hidden_size
    assert call(_cfg(), cu=1) == -1                      # packed mode needs both cu_seqlens and tok_src
    assert call(_cfg(), cu=1, tok=1, n=17) == -1         # more packed rows than B * L
    assert call(_cfg(), ws_bytes=16) == -3               # workspace too small
    assert call(_cfg(), B=0) == 0                        # empty batch: no-op
