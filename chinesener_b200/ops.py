"""Thin functional wrappers over the C-ABI (one per exported kernel family).

Each function checks devices/dtypes/contiguity, allocates outputs with torch, and forwards raw
pointers + the current CUDA stream to libner_b200.so.  Nothing here computes on the CPU.
"""
import torch

from . import _lib
from ._lib import NerB200Error, check, lib, ptr, require_cuda, stream

EPI_F32, EPI_BF16, EPI_GELU_TANH_BF16, EPI_GELU_ERF_BF16, EPI_RELU_BF16, EPI_RES_F32, EPI_RES_RELU_F32 = range(7)
EPI_DIAG_DISCARD = 99
EPI_GELU_TANH_E4M3, EPI_GELU_ERF_E4M3 = 7, 8   # ner_gemm_e4m3 only: GELU -> e4m3 with 1 x 128 block scales
E4M3 = torch.float8_e4m3fn
TILE_2CTA_128, TILE_2CTA_256 = 1128, 1256   # CTA-pair (cta_group::2) tiles of ner_gemm_bf16
TILE_SK_128, TILE_SK_256 = 2128, 2256       # stream-K scheduling of 128 x {128,256} tiles
TILE_AUTO_THROUGHPUT = 3000                 # auto, preferring the tile with the best FLOP rate (multi-stream serving)
DEFAULT_TILE = 0                            # what gemm_bf16(tile_n=None) passes; predict_iter(streams>1) switches it


def _i32(t):
    return t if t.dtype == torch.int32 else t.to(torch.int32)


# --------------------------------------------------------------------------- CRF
MAX_TAGS = 32        # K of the K-specialised CRF kernels (NER_MAX_TAGS); ops.crf_* send larger K to the wide ones
MAX_TAGS_WIDE = 128  # NER_MAX_TAGS_WIDE


def _wide(K, wide):
    """Whether a CRF call runs the wide-tag-set kernels (ner_crf_wide_*): always past MAX_TAGS; wide=True forces them
    for any K (the tests pin them to the K-specialised kernels, the bench compares the two)."""
    return K > MAX_TAGS or bool(wide)


def crf_viterbi(logits, seq_len, trans, return_score=False, wide=None):
    """tf.contrib.crf.crf_decode (reference tools/layer.py:140).  -> tags [B,L] int32 (+ best_score [B]).
    K <= 32: ner_crf_viterbi; K <= 128 (or wide=True): ner_crf_wide_viterbi with its backpointer workspace."""
    require_cuda(logits, seq_len, trans)
    assert logits.dtype == torch.float32 and trans.dtype == torch.float32
    B, L, K = logits.shape
    assert trans.shape == (K, K)
    seq_len = _i32(seq_len)
    dev = logits.device
    tags = torch.empty((B, L), dtype=torch.int32, device=dev)
    score = torch.empty((B,), dtype=torch.float32, device=dev) if return_score else None
    if _wide(K, wide):
        nbytes = int(lib().ner_crf_wide_viterbi_workspace_bytes(B, L, K))
        ws = torch.empty((max(nbytes, 16),), dtype=torch.uint8, device=dev)
        check(lib().ner_crf_wide_viterbi(ptr(logits), ptr(seq_len), ptr(trans), ptr(tags), ptr(score), ptr(ws), nbytes,
                                         B, L, K, stream()))
    else:
        check(lib().ner_crf_viterbi(ptr(logits), ptr(seq_len), ptr(trans), ptr(tags), ptr(score), B, L, K, stream()))
    return (tags, score) if return_score else tags


NBEST_MAX = 16                                   # largest n of crf_viterbi_nbest


def crf_viterbi_nbest(logits, seq_len, trans, n):
    """N-best tf.contrib.crf.crf_decode (ner_crf_viterbi_nbest) -> (tags [B,n,L] int32, scores [B,n] f32, counts [B]
    int32).  Rank 0 is crf_viterbi's path and best_score; ranks past counts[b] are zero tags with score -inf."""
    require_cuda(logits, seq_len, trans)
    assert logits.dtype == torch.float32 and trans.dtype == torch.float32
    B, L, K = logits.shape
    assert trans.shape == (K, K)
    n = int(n)
    seq_len = _i32(seq_len)
    dev = logits.device
    tags = torch.empty((B, n, L), dtype=torch.int32, device=dev)
    scores = torch.empty((B, n), dtype=torch.float32, device=dev)
    counts = torch.zeros((B,), dtype=torch.int32, device=dev)
    nbytes = int(lib().ner_crf_viterbi_nbest_workspace_bytes(B, L, K, n))
    ws = torch.empty((max(nbytes, 16),), dtype=torch.uint8, device=dev)
    check(lib().ner_crf_viterbi_nbest(ptr(logits), ptr(seq_len), ptr(trans), n, ptr(tags), ptr(scores), ptr(counts),
                                      ptr(ws), nbytes, B, L, K, stream()))
    return tags, scores, counts


def crf_loglik_fwd(logits, tags, seq_len, trans, want_alpha=False, exact=False, wide=None):
    """tf.contrib.crf.crf_log_likelihood forward (reference tools/layer.py:122). -> ll [B], logz [B], alpha|None.
    K <= 32: ner_crf_loglik_fwd; K <= 128 (or wide=True): ner_crf_wide_loglik_fwd."""
    require_cuda(logits, tags, seq_len, trans)
    assert logits.dtype == torch.float32 and trans.dtype == torch.float32
    B, L, K = logits.shape
    tags, seq_len = _i32(tags), _i32(seq_len)
    ll = torch.empty((B,), dtype=torch.float32, device=logits.device)
    logz = torch.empty((B,), dtype=torch.float32, device=logits.device)
    alpha = torch.empty((B, L, K), dtype=torch.float32, device=logits.device) if want_alpha else None
    fn = lib().ner_crf_wide_loglik_fwd if _wide(K, wide) else lib().ner_crf_loglik_fwd
    check(fn(ptr(logits), ptr(tags), ptr(seq_len), ptr(trans), ptr(ll), ptr(logz), ptr(alpha), B, L, K,
             1 if exact else 0, stream()))
    return ll, logz, alpha


# --------------------------------------------------------------------------- dense (wgmma)
def gemm_bf16(a, wt, bias=None, residual=None, epilogue=EPI_BF16, tile_n=None, out=None):
    """out[M,N] = epilogue(a[M,K] @ wt[N,K]^T + bias).  a, wt bf16; see ner_gemm_bf16.  tile_n None = DEFAULT_TILE."""
    if tile_n is None:
        tile_n = DEFAULT_TILE
    require_cuda(a, wt, bias, residual, out)
    assert a.dtype == torch.bfloat16 and wt.dtype == torch.bfloat16
    M, K = a.shape
    N, K2 = wt.shape
    assert K == K2
    odt = torch.float32 if epilogue in (EPI_F32, EPI_RES_F32, EPI_RES_RELU_F32) else torch.bfloat16
    if out is None:
        out = torch.empty((M, N), dtype=odt, device=a.device)
    assert out.dtype == odt and out.shape == (M, N)
    if bias is not None:
        assert bias.dtype == torch.float32 and bias.numel() == N
    if residual is not None:
        assert residual.dtype == torch.float32 and residual.shape == (M, N)
    hook = _lib._HOOK
    if hook is not None:
        with hook("gemm_bf16", 2.0 * M * N * K):
            check(lib().ner_gemm_bf16(ptr(a), ptr(wt), ptr(bias), ptr(residual), ptr(out), M, N, K, epilogue, tile_n, stream()))
    else:
        check(lib().ner_gemm_bf16(ptr(a), ptr(wt), ptr(bias), ptr(residual), ptr(out), M, N, K, epilogue, tile_n, stream()))
    return out


def pack_weight_bf16(w_kn):
    """TF dense kernel [K,N] f32 -> bf16 [N,K] (B operand layout of gemm_bf16)."""
    require_cuda(w_kn)
    assert w_kn.dtype == torch.float32 and w_kn.dim() == 2
    K, N = w_kn.shape
    out = torch.empty((N, K), dtype=torch.bfloat16, device=w_kn.device)
    check(lib().ner_pack_weight_bf16(ptr(w_kn), ptr(out), K, N, stream()))
    return out


def gemm_e4m3(a, a_scale, wt, w_scale, bias=None, epilogue=EPI_BF16, out=None, out_scale=None):
    """FP8 dense layer with block scales (ner_gemm_e4m3): a e4m3 [M,K] + a_scale f32 [M, K/128], wt e4m3 [N,K] + w_scale
    f32 [N].  EPI_BF16 -> bf16 [M,N]; EPI_GELU_*_E4M3 -> (e4m3 [M,N], f32 block scales [M, N/128])."""
    require_cuda(a, a_scale, wt, w_scale, bias, out, out_scale)
    assert a.dtype == E4M3 and wt.dtype == E4M3 and a_scale.dtype == torch.float32 and w_scale.dtype == torch.float32
    M, K = a.shape
    N, K2 = wt.shape
    assert K == K2 and w_scale.numel() == N and a_scale.shape == (M, K // 128)
    if bias is not None:
        assert bias.dtype == torch.float32 and bias.numel() == N
    q_out = epilogue in (EPI_GELU_TANH_E4M3, EPI_GELU_ERF_E4M3)
    if out is None:
        out = torch.empty((M, N), dtype=E4M3 if q_out else torch.bfloat16, device=a.device)
    if q_out and out_scale is None:
        out_scale = torch.empty((M, N // 128), dtype=torch.float32, device=a.device)
    hook = _lib._HOOK
    args = (ptr(a), ptr(a_scale), ptr(wt), ptr(w_scale), ptr(bias), ptr(out), ptr(out_scale), M, N, K, epilogue, stream())
    if hook is not None:
        with hook("gemm_e4m3", 2.0 * M * N * K):
            check(lib().ner_gemm_e4m3(*args))
    else:
        check(lib().ner_gemm_e4m3(*args))
    return (out, out_scale) if q_out else out


def quantize_weight_e4m3(w_kn):
    """TF dense kernel [K,N] f32 -> (e4m3 [N,K], f32 per-channel scales [N]): the B operand of gemm_e4m3."""
    require_cuda(w_kn)
    assert w_kn.dtype == torch.float32 and w_kn.dim() == 2
    K, N = w_kn.shape
    q = torch.empty((N, K), dtype=E4M3, device=w_kn.device)
    sc = torch.empty((N,), dtype=torch.float32, device=w_kn.device)
    check(lib().ner_quantize_weight_e4m3(ptr(w_kn), ptr(q), ptr(sc), K, N, stream()))
    return q, sc


def cast_bf16(x):
    require_cuda(x)
    assert x.dtype == torch.float32
    out = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
    check(lib().ner_cast_bf16(ptr(x), ptr(out), x.numel(), stream()))
    return out


def dense_small_n(x, w, bias=None, row_map=None, out=None):
    """tf.layers.dense(units=label_size): x [M,F] (f32|bf16) @ w [F,N] f32 + bias -> f32 [M,N], N <= 32.
    row_map [M] i32 scatters input row r to out[row_map[r]] (packed -> padded); `out` then must be given."""
    require_cuda(x, w, bias, row_map, out)
    assert w.dtype == torch.float32 and x.dtype in (torch.float32, torch.bfloat16)
    M, F = x.shape
    F2, N = w.shape
    assert F == F2
    if out is None:
        assert row_map is None
        out = torch.empty((M, N), dtype=torch.float32, device=x.device)
    check(lib().ner_dense_small_n(ptr(x), 1 if x.dtype == torch.bfloat16 else 0, ptr(w), ptr(bias), ptr(out), M, F, N,
                                  ptr(row_map), stream()))
    return out


def seq_pack_plan(mask):
    """prefix mask [B,L] -> (cu_seqlens [B+1] i32, tok_src [B*L] i32) on the device."""
    require_cuda(mask)
    B, L = mask.shape
    mask = _i32(mask)
    cu = torch.empty((B + 1,), dtype=torch.int32, device=mask.device)
    tok_src = torch.empty((B * L,), dtype=torch.int32, device=mask.device)
    check(lib().ner_seq_pack_plan(ptr(mask), ptr(cu), ptr(tok_src), B, L, stream()))
    return cu, tok_src


# --------------------------------------------------------------------------- BERT pieces
def bert_embed_ln(word_emb, type_emb, pos_emb, gamma, beta, ids, seg, eps=1e-12, want_f32=True, want_bf16=True,
                  tok_src=None, n_packed=0):
    """Padded mode: B*L output rows.  Packed mode (tok_src, n_packed): n_packed rows."""
    require_cuda(word_emb, type_emb, pos_emb, gamma, beta, ids, seg, tok_src)
    B, L = ids.shape
    V, H = word_emb.shape
    ids = _i32(ids)
    seg = None if seg is None else _i32(seg)
    rows = n_packed if tok_src is not None else B * L
    of = torch.empty((rows, H), dtype=torch.float32, device=ids.device) if want_f32 else None
    ob = torch.empty((rows, H), dtype=torch.bfloat16, device=ids.device) if want_bf16 else None
    check(lib().ner_bert_embed_ln(ptr(word_emb), ptr(type_emb), ptr(pos_emb), ptr(gamma), ptr(beta), ptr(ids), ptr(seg),
                                  ptr(of), ptr(ob), B, L, H, V, type_emb.shape[0], pos_emb.shape[0], eps, ptr(tok_src),
                                  n_packed, stream()))
    return of, ob


def layernorm(y, gamma, beta, residual=None, eps=1e-12, want_f32=True, want_bf16=True, keep_prob=1.0, seed=0):
    """LN(dropout(y) + residual); keep_prob < 1 fuses BertModel's hidden dropout (training)."""
    require_cuda(y, gamma, beta, residual)
    assert y.dtype in (torch.float32, torch.bfloat16)
    M, H = y.shape
    of = torch.empty((M, H), dtype=torch.float32, device=y.device) if want_f32 else None
    ob = torch.empty((M, H), dtype=torch.bfloat16, device=y.device) if want_bf16 else None
    check(lib().ner_layernorm_dropout(ptr(y), 1 if y.dtype == torch.bfloat16 else 0, ptr(residual), ptr(gamma), ptr(beta),
                                      ptr(of), ptr(ob), M, H, eps, float(keep_prob), int(seed) & 0xFFFFFFFFFFFFFFFF, stream()))
    return of, ob


def bert_embed_ln_e4m3(word_emb, type_emb, pos_emb, gamma, beta, ids, seg, eps=1e-12, tok_src=None, n_packed=0):
    """bert_embed_ln writing f32 + the e4m3 copy with 1 x 128 block scales -> (f32 [rows,H], e4m3 [rows,H], f32 [rows,H/128])."""
    require_cuda(word_emb, type_emb, pos_emb, gamma, beta, ids, seg, tok_src)
    B, L = ids.shape
    V, H = word_emb.shape
    ids = _i32(ids)
    seg = None if seg is None else _i32(seg)
    rows = n_packed if tok_src is not None else B * L
    of = torch.empty((rows, H), dtype=torch.float32, device=ids.device)
    oq = torch.empty((rows, H), dtype=E4M3, device=ids.device)
    osc = torch.empty((rows, H // 128), dtype=torch.float32, device=ids.device)
    check(lib().ner_bert_embed_ln_e4m3(ptr(word_emb), ptr(type_emb), ptr(pos_emb), ptr(gamma), ptr(beta), ptr(ids), ptr(seg),
                                       ptr(of), None, ptr(oq), ptr(osc), B, L, H, V, type_emb.shape[0], pos_emb.shape[0], eps,
                                       ptr(tok_src), n_packed, stream()))
    return of, oq, osc


def layernorm_e4m3(y, gamma, beta, residual=None, eps=1e-12):
    """LN(y + residual) -> (f32 [M,H], e4m3 [M,H], f32 block scales [M, H/128])."""
    require_cuda(y, gamma, beta, residual)
    assert y.dtype in (torch.float32, torch.bfloat16)
    M, H = y.shape
    of = torch.empty((M, H), dtype=torch.float32, device=y.device)
    oq = torch.empty((M, H), dtype=E4M3, device=y.device)
    osc = torch.empty((M, H // 128), dtype=torch.float32, device=y.device)
    check(lib().ner_layernorm_e4m3(ptr(y), 1 if y.dtype == torch.bfloat16 else 0, ptr(residual), ptr(gamma), ptr(beta),
                                   ptr(of), None, ptr(oq), ptr(osc), M, H, eps, stream()))
    return of, oq, osc


def bert_attention(qkv, mask, B, L, num_heads, head_dim=64, scale=None, mask_add=-10000.0, cu_seqlens=None, keep_prob=1.0,
                   seed=0):
    """Padded mode: qkv [B*L, 3HD] + mask.  Packed mode: qkv [T, 3HD] + cu_seqlens [B+1] (L = max length).
    keep_prob < 1: attention_probs dropout (training)."""
    require_cuda(qkv, mask, cu_seqlens)
    assert qkv.dtype == torch.bfloat16 and qkv.shape[1] == 3 * num_heads * head_dim
    assert cu_seqlens is not None or qkv.shape[0] == B * L
    mask = None if mask is None else _i32(mask)
    ctx = torch.empty((qkv.shape[0], num_heads * head_dim), dtype=torch.bfloat16, device=qkv.device)
    if scale is None:
        scale = 1.0 / (head_dim ** 0.5)
    check(lib().ner_bert_attention(ptr(qkv), ptr(mask), ptr(ctx), B, L, num_heads, head_dim, scale, mask_add,
                                   ptr(cu_seqlens), int(qkv.shape[0]), float(keep_prob), int(seed) & 0xFFFFFFFFFFFFFFFF, stream()))
    return ctx


# --------------------------------------------------------------------------- BiLSTM
def bilstm_recurrence(xproj, wh_fw, wh_bw, seq_len, B, L, H, activation="tanh", forget_bias=1.0, cu_seqlens=None,
                      save_for_backward=False, keep_prob=1.0, seed=0):
    """-> out [B,L,2H]; with save_for_backward also (gates [B*L,8H], cstate [B,L,2H], hstate [B,L,2H]) for
    bilstm_recurrence_bwd.  keep_prob < 1: DropoutWrapper output/state dropout (training)."""
    require_cuda(xproj, wh_fw, wh_bw, seq_len, cu_seqlens)
    assert xproj.dtype == torch.float32 and xproj.shape[1] == 8 * H
    assert cu_seqlens is not None or xproj.shape[0] == B * L
    assert wh_fw.shape == (H, 4 * H) and wh_bw.shape == (H, 4 * H)
    act = {"tanh": 0, "relu": 1}[activation]
    out = torch.empty((B, L, 2 * H), dtype=torch.float32, device=xproj.device)
    gates = cst = hst = None
    if save_for_backward:
        assert cu_seqlens is None, "training runs on the padded layout"
        gates = torch.zeros((B * L, 8 * H), dtype=torch.float32, device=xproj.device)
        cst = torch.zeros((B, L, 2 * H), dtype=torch.float32, device=xproj.device)
        hst = torch.zeros((B, L, 2 * H), dtype=torch.float32, device=xproj.device)
    check(lib().ner_bilstm_recurrence(ptr(xproj), ptr(wh_fw), ptr(wh_bw), ptr(_i32(seq_len)), ptr(out), B, L, H, act,
                                      forget_bias, ptr(cu_seqlens), ptr(gates), ptr(cst), ptr(hst), float(keep_prob),
                                      int(seed) & 0xFFFFFFFFFFFFFFFF, stream()))
    return (out, gates, cst, hst) if save_for_backward else out


def bilstm_recurrence_bwd(d_out, gates, cstate, wh_fw, wh_bw, seq_len, B, L, H, activation="tanh", keep_prob=1.0, seed=0):
    """-> d_xproj [B*L, 8H] f32 (gradient of the hoisted input projection)."""
    require_cuda(d_out, gates, cstate, wh_fw, wh_bw, seq_len)
    assert d_out.shape == (B, L, 2 * H) and d_out.dtype == torch.float32
    act = {"tanh": 0, "relu": 1}[activation]
    d_xproj = torch.empty((B * L, 8 * H), dtype=torch.float32, device=d_out.device)
    check(lib().ner_bilstm_recurrence_bwd(ptr(d_out), ptr(gates), ptr(cstate), ptr(wh_fw), ptr(wh_bw), ptr(_i32(seq_len)),
                                          ptr(d_xproj), B, L, H, act, float(keep_prob), int(seed) & 0xFFFFFFFFFFFFFFFF,
                                          stream()))
    return d_xproj


# --------------------------------------------------------------------------- BiGRU
def bigru_recurrence(xproj, wh_fw, wh_bw, seq_len, B, L, H, activation="tanh", cu_seqlens=None, save_for_backward=False,
                     keep_prob=1.0, seed=0):
    """GRUCell recurrence of both directions: xproj [rows, >= 6H] (extra columns are GEMM padding), wh_* [H, 3H] (columns r, u, c) -> out [B,L,2H]; with
    save_for_backward also (gates [B*L,6H] = r, u, c; hstate [B,L,2H] carried h; rh [B,L,2H] = r ⊙ h_prev) for
    bigru_recurrence_bwd.  keep_prob < 1: DropoutWrapper output/state dropout (training)."""
    require_cuda(xproj, wh_fw, wh_bw, seq_len, cu_seqlens)
    assert xproj.dtype == torch.float32 and xproj.shape[1] >= 6 * H
    assert cu_seqlens is not None or xproj.shape[0] == B * L
    assert wh_fw.shape == (H, 3 * H) and wh_bw.shape == (H, 3 * H)
    act = {"tanh": 0, "relu": 1}[activation]
    out = torch.empty((B, L, 2 * H), dtype=torch.float32, device=xproj.device)
    gates = hst = rh = None
    if save_for_backward:
        assert cu_seqlens is None, "training runs on the padded layout"
        gates = torch.zeros((B * L, 6 * H), dtype=torch.float32, device=xproj.device)
        hst = torch.zeros((B, L, 2 * H), dtype=torch.float32, device=xproj.device)
        rh = torch.zeros((B, L, 2 * H), dtype=torch.float32, device=xproj.device)
    check(lib().ner_bigru_recurrence(ptr(xproj), ptr(wh_fw), ptr(wh_bw), ptr(_i32(seq_len)), ptr(out), B, L, H, xproj.shape[1],
                                     act, ptr(cu_seqlens), ptr(gates), ptr(hst), ptr(rh), float(keep_prob),
                                     int(seed) & 0xFFFFFFFFFFFFFFFF, stream()))
    return (out, gates, hst, rh) if save_for_backward else out


def bigru_recurrence_bwd(d_out, gates, hstate, wh_fw, wh_bw, seq_len, B, L, H, activation="tanh", keep_prob=1.0, seed=0):
    """-> d_xproj [B*L, 6H] f32 (columns da_r, da_u, da_c per direction: the gradient of the hoisted input projection)."""
    require_cuda(d_out, gates, hstate, wh_fw, wh_bw, seq_len)
    assert d_out.shape == (B, L, 2 * H) and d_out.dtype == torch.float32
    assert gates.shape == (B * L, 6 * H) and hstate.shape == (B, L, 2 * H)
    act = {"tanh": 0, "relu": 1}[activation]
    d_xproj = torch.empty((B * L, 6 * H), dtype=torch.float32, device=d_out.device)
    check(lib().ner_bigru_recurrence_bwd(ptr(d_out), ptr(gates), ptr(hstate), ptr(wh_fw), ptr(wh_bw), ptr(_i32(seq_len)),
                                         ptr(d_xproj), B, L, H, act, float(keep_prob), int(seed) & 0xFFFFFFFFFFFFFFFF,
                                         stream()))
    return d_xproj


# --------------------------------------------------------------------------- Lattice LSTM
def lattice_recurrence(xproj, wproj, lat_len, wrec_fw, wrec_bw, wac_fw, wac_bw, seq_len, B, L, H, Kw,
                       save_for_backward=False):
    """Lattice LSTM recurrence of both directions (ner_lattice_recurrence): xproj [B*L, 8H], wproj [B*L*Kw, 6H],
    lat_len int32 [B, L*Kw], wrec_* [H, 6H], wac_* [H, H] -> out [B, L, 2H]; with save_for_backward also the dict of
    saved tensors lattice_recurrence_bwd reads (gates, cstate, norm, wgates, cw, aw, hw)."""
    require_cuda(xproj, wproj, lat_len, wrec_fw, wrec_bw, wac_fw, wac_bw, seq_len)
    assert xproj.dtype == torch.float32 and xproj.shape == (B * L, 8 * H)
    assert wproj.dtype == torch.float32 and wproj.shape == (B * L * Kw, 6 * H)
    assert lat_len.dtype == torch.int32 and lat_len.numel() == B * L * Kw
    assert wrec_fw.shape == (H, 6 * H) and wrec_bw.shape == (H, 6 * H) and wac_fw.shape == (H, H) and wac_bw.shape == (H, H)
    dev = xproj.device
    out = torch.empty((B, L, 2 * H), dtype=torch.float32, device=dev)
    sv = None
    if save_for_backward:
        sv = dict(gates=torch.zeros((B * L, 6 * H), dtype=torch.float32, device=dev),
                  cstate=torch.zeros((B, L, 2 * H), dtype=torch.float32, device=dev),
                  norm=torch.zeros((B, L, 2 * H), dtype=torch.float32, device=dev),
                  wgates=torch.zeros((B * L * Kw, 6 * H), dtype=torch.float32, device=dev),
                  cw=torch.zeros((B * L * Kw, 2 * H), dtype=torch.float32, device=dev),
                  aw=torch.zeros((B * L * Kw, 2 * H), dtype=torch.float32, device=dev),
                  hw=torch.zeros((B * L * Kw, 2 * H), dtype=torch.float32, device=dev))
    s = sv or {}
    check(lib().ner_lattice_recurrence(ptr(xproj), ptr(wproj), ptr(lat_len), ptr(wrec_fw), ptr(wrec_bw), ptr(wac_fw),
                                       ptr(wac_bw), ptr(_i32(seq_len)), ptr(out), B, L, H, Kw, ptr(s.get('gates')),
                                       ptr(s.get('cstate')), ptr(s.get('norm')), ptr(s.get('wgates')), ptr(s.get('cw')),
                                       ptr(s.get('aw')), ptr(s.get('hw')), stream()))
    return (out, sv) if save_for_backward else out


def lattice_recurrence_bwd(d_out, saved, lat_len, wrec_fw, wrec_bw, wac_fw, wac_bw, seq_len, B, L, H, Kw):
    """-> (d_xproj [B*L, 8H], d_wproj [B*L*Kw, 6H], d_alpha [B*L*Kw, 2H]): the gradients of the two hoisted projections
    and of each word's alpha pre-activation (zero on empty slots)."""
    require_cuda(d_out, lat_len, wrec_fw, wrec_bw, wac_fw, wac_bw, seq_len)
    assert d_out.shape == (B, L, 2 * H) and d_out.dtype == torch.float32
    dev = d_out.device
    d_xproj = torch.empty((B * L, 8 * H), dtype=torch.float32, device=dev)
    d_wproj = torch.zeros((B * L * Kw, 6 * H), dtype=torch.float32, device=dev)
    d_alpha = torch.zeros((B * L * Kw, 2 * H), dtype=torch.float32, device=dev)
    s = saved
    check(lib().ner_lattice_recurrence_bwd(ptr(d_out), ptr(s['gates']), ptr(s['cstate']), ptr(s['norm']), ptr(s['wgates']),
                                           ptr(s['cw']), ptr(s['aw']), ptr(lat_len), ptr(wrec_fw), ptr(wrec_bw),
                                           ptr(wac_fw), ptr(wac_bw), ptr(_i32(seq_len)), ptr(d_xproj), ptr(d_wproj),
                                           ptr(d_alpha), B, L, H, Kw, stream()))
    return d_xproj, d_wproj, d_alpha


# --------------------------------------------------------------------------- SoftLexicon
def softlexicon_pool(table, ids, weights, G=4, S=10, out=None):
    """ids/weights [..., G*S] -> [..., G*E]; `out` may be a wider [n_tok, >=G*E] buffer (concat target)."""
    require_cuda(table, ids, weights, out)
    assert table.dtype == torch.float32 and weights.dtype == torch.float32
    V, E = table.shape
    lead = ids.shape[:-1]
    assert ids.shape[-1] == G * S and weights.shape == ids.shape
    n_tok = ids.numel() // (G * S)
    if out is None:
        out = torch.empty((*lead, G * E), dtype=torch.float32, device=table.device)
    ld = out.shape[-1]
    check(lib().ner_softlexicon_pool_fwd(ptr(table), ptr(_i32(ids)), ptr(weights), ptr(out), n_tok, G, S, E, V, ld,
                                         stream()))
    return out


def embedding_lookup(table, ids, out=None, col_offset=0):
    """tf.nn.embedding_lookup into out[..., col_offset:col_offset+E] (out row-major [n_tok, ld])."""
    require_cuda(table, ids, out)
    assert table.dtype == torch.float32
    V, E = table.shape
    n_tok = ids.numel()
    if out is None:
        out = torch.empty((*ids.shape, E), dtype=torch.float32, device=table.device)
    ld = out.shape[-1]
    assert col_offset + E <= ld
    check(lib().ner_embedding_lookup(ptr(table), ptr(_i32(ids)), out.data_ptr() + 4 * col_offset, n_tok, E, V, ld, stream()))
    return out


def cast_pad_bf16(x2d, Dp):
    """f32 [M,D] -> bf16 [M,Dp] zero padded."""
    require_cuda(x2d)
    assert x2d.dtype == torch.float32 and x2d.dim() == 2
    M, D = x2d.shape
    out = torch.empty((M, Dp), dtype=torch.bfloat16, device=x2d.device)
    check(lib().ner_cast_pad_bf16(ptr(x2d), ptr(out), M, D, Dp, D, stream()))
    return out


def softlexicon_pool_bwd(d_table, ids, weights, d_out, G=4, S=10):
    require_cuda(d_table, ids, weights, d_out)
    V, E = d_table.shape
    n_tok = ids.numel() // (G * S)
    check(lib().ner_softlexicon_pool_bwd(ptr(d_table), ptr(_i32(ids)), ptr(weights), ptr(d_out), n_tok, G, S, E, V,
                                         stream()))
    return d_table


# --------------------------------------------------------------------------- small word-enhance tables
def multihot_embed(table, weights, out=None, col_offset=0):
    """weights [..., V] @ table [V, E] (ner_multihot_embed_fwd) into out[..., col_offset:col_offset+E]."""
    require_cuda(table, weights, out)
    assert table.dtype == torch.float32 and weights.dtype == torch.float32
    V, E = table.shape
    assert weights.shape[-1] == V
    n_tok = weights.numel() // V
    if out is None:
        out = torch.empty((*weights.shape[:-1], E), dtype=torch.float32, device=table.device)
    ld = out.shape[-1]
    assert col_offset + E <= ld and out.numel() == n_tok * ld
    check(lib().ner_multihot_embed_fwd(ptr(table), ptr(weights), out.data_ptr() + 4 * col_offset, n_tok, V, E, ld, stream()))
    return out


_small_table_scratch = {}


def small_table_grad(d_table, d_out, ids=None, weights=None, col_offset=0):
    """d_table [V, E] += the gradient of embedding_lookup(table, ids) (one-hot) or multihot_embed(table, weights),
    read from d_out[..., col_offset:col_offset+E] (d_out row-major [n_tok, ld]).  Deterministic (ner_small_table_grad)."""
    require_cuda(d_table, d_out, ids, weights)
    assert (ids is None) != (weights is None)
    assert d_table.dtype == torch.float32 and d_out.dtype == torch.float32
    V, E = d_table.shape
    n_tok = ids.numel() if ids is not None else weights.numel() // V
    ld = d_out.shape[-1]
    assert col_offset + E <= ld and d_out.numel() == n_tok * ld
    need = int(lib().ner_small_table_grad_scratch_floats(V, E))
    key = (d_table.device.index, stream())
    scratch = _small_table_scratch.get(key)
    if scratch is None or scratch.numel() < need:
        scratch = _small_table_scratch[key] = torch.empty(max(need, 1), dtype=torch.float32, device=d_table.device)
    check(lib().ner_small_table_grad(ptr(d_table), ptr(None if ids is None else _i32(ids)), ptr(weights),
                                     d_out.data_ptr() + 4 * col_offset, n_tok, V, E, ld, ptr(scratch), stream()))
    return d_table


def crf_loglik_bwd(logits, tags, seq_len, trans, alpha, logz, d_ll=None, scale=1.0, wide=None):
    """-> d_logits [B,L,K], d_trans [K,K] for g_b = (d_ll|1) * scale.  K <= 32: ner_crf_loglik_bwd; K <= 128 (or
    wide=True): ner_crf_wide_loglik_bwd."""
    require_cuda(logits, tags, seq_len, trans, alpha, logz, d_ll)
    B, L, K = logits.shape
    assert all(t.dtype == torch.float32 for t in (logits, trans, alpha, logz) + ((d_ll,) if d_ll is not None else ()))
    assert trans.shape == (K, K) and alpha.shape == (B, L, K) and logz.shape == (B,)
    assert d_ll is None or d_ll.shape == (B,)
    d_logits = torch.empty_like(logits)
    d_trans = torch.zeros_like(trans)
    fn = lib().ner_crf_wide_loglik_bwd if _wide(K, wide) else lib().ner_crf_loglik_bwd
    check(fn(ptr(logits), ptr(_i32(tags)), ptr(_i32(seq_len)), ptr(trans), ptr(alpha), ptr(logz), ptr(d_ll), scale,
             ptr(d_logits), ptr(d_trans), B, L, K, stream()))
    return d_logits, d_trans


def crf_partial_loglik_fwd(logits, label_mask, seq_len, trans, want_alpha=False, exact=False):
    """Partial-annotation CRF log-likelihood (ner_crf_partial_loglik_fwd): label_mask [B,L] int32 bitmasks of the
    allowed tags. -> ll [B], logz [B,2] (logZ_A, logZ), alpha [2,B,L,K] | None."""
    require_cuda(logits, label_mask, seq_len, trans)
    assert logits.dtype == torch.float32 and trans.dtype == torch.float32
    B, L, K = logits.shape
    assert trans.shape == (K, K) and label_mask.shape == (B, L)
    label_mask, seq_len = _i32(label_mask), _i32(seq_len)
    ll = torch.empty((B,), dtype=torch.float32, device=logits.device)
    logz = torch.empty((B, 2), dtype=torch.float32, device=logits.device)
    alpha = torch.empty((2, B, L, K), dtype=torch.float32, device=logits.device) if want_alpha else None
    check(lib().ner_crf_partial_loglik_fwd(ptr(logits), ptr(label_mask), ptr(seq_len), ptr(trans), ptr(ll), ptr(logz),
                                           ptr(alpha), B, L, K, 1 if exact else 0, stream()))
    return ll, logz, alpha


def crf_partial_loglik_bwd(logits, label_mask, seq_len, trans, alpha, logz, d_ll=None, scale=1.0):
    """-> d_logits [B,L,K], d_trans [K,K] of sum_b g_b ll_b, g_b = (d_ll|1) * scale (ner_crf_partial_loglik_bwd)."""
    require_cuda(logits, label_mask, seq_len, trans, alpha, logz, d_ll)
    B, L, K = logits.shape
    assert all(t.dtype == torch.float32 for t in (logits, trans, alpha, logz) + ((d_ll,) if d_ll is not None else ()))
    assert trans.shape == (K, K) and alpha.shape == (2, B, L, K) and logz.shape == (B, 2)
    assert label_mask.shape == (B, L) and (d_ll is None or d_ll.shape == (B,))
    d_logits = torch.empty_like(logits)
    d_trans = torch.zeros_like(trans)
    check(lib().ner_crf_partial_loglik_bwd(ptr(logits), ptr(_i32(label_mask)), ptr(_i32(seq_len)), ptr(trans),
                                           ptr(alpha), ptr(logz), ptr(d_ll), scale, ptr(d_logits), ptr(d_trans),
                                           B, L, K, stream()))
    return d_logits, d_trans


def crf_distill_fwd(t_logits, t_trans, s_logits, s_trans, seq_len, temperature=1.0, exact=False):
    """Forward half of CRF-to-CRF distillation at temperature tau (ner_crf_distill_fwd): teacher and student share
    [B,L,K].  -> logz [B,2] (logZ_T, logZ_S of the tau-scaled CRFs), alpha [2,B,L,K] for crf_distill_bwd."""
    require_cuda(t_logits, t_trans, s_logits, s_trans, seq_len)
    assert all(t.dtype == torch.float32 for t in (t_logits, t_trans, s_logits, s_trans))
    B, L, K = s_logits.shape
    assert t_logits.shape == (B, L, K) and t_trans.shape == (K, K) and s_trans.shape == (K, K)
    t_logits, s_logits = t_logits.contiguous(), s_logits.contiguous()
    logz = torch.empty((B, 2), dtype=torch.float32, device=s_logits.device)
    alpha = torch.empty((2, B, L, K), dtype=torch.float32, device=s_logits.device)
    check(lib().ner_crf_distill_fwd(ptr(t_logits), ptr(t_trans.contiguous()), ptr(s_logits), ptr(s_trans.contiguous()),
                                    ptr(_i32(seq_len)), 1.0 / float(temperature), ptr(logz), ptr(alpha), B, L, K,
                                    1 if exact else 0, stream()))
    return logz, alpha


def crf_distill_bwd(t_logits, t_trans, s_logits, s_trans, seq_len, alpha, logz, temperature=1.0, d_kl=None, scale=1.0,
                    exact=False):
    """-> kl [B] (KL(teacher || student) over all paths at temperature tau), d_s_logits [B,L,K], d_s_trans [K,K] of
    sum_b g_b KL_b, g_b = (d_kl|1) * scale (ner_crf_distill_bwd).  The teacher gets no gradient."""
    require_cuda(t_logits, t_trans, s_logits, s_trans, seq_len, alpha, logz, d_kl)
    B, L, K = s_logits.shape
    assert all(t.dtype == torch.float32 for t in (t_logits, t_trans, s_logits, s_trans, alpha, logz)
               + ((d_kl,) if d_kl is not None else ()))
    assert t_logits.shape == (B, L, K) and alpha.shape == (2, B, L, K) and logz.shape == (B, 2)
    assert d_kl is None or d_kl.shape == (B,)
    t_logits, s_logits = t_logits.contiguous(), s_logits.contiguous()
    kl = torch.empty((B,), dtype=torch.float32, device=s_logits.device)
    d_logits = torch.empty_like(s_logits)
    d_trans = torch.zeros_like(s_trans)
    check(lib().ner_crf_distill_bwd(ptr(t_logits), ptr(t_trans.contiguous()), ptr(s_logits), ptr(s_trans.contiguous()),
                                    ptr(_i32(seq_len)), 1.0 / float(temperature), ptr(alpha), ptr(logz),
                                    ptr(None if d_kl is None else d_kl.contiguous()), scale, ptr(kl), ptr(d_logits),
                                    ptr(d_trans), B, L, K, 1 if exact else 0, stream()))
    return kl, d_logits, d_trans


# --------------------------------------------------------------------------- fp32-accurate dense (split bf16)
def split_bf16(x2d, Dp=None):
    """f32 [M,D] -> (hi, lo) bf16 [M,Dp] with hi + lo ~= x to 2^-17."""
    require_cuda(x2d)
    assert x2d.dtype == torch.float32 and x2d.dim() == 2 and x2d.stride(1) == 1
    M, D = x2d.shape
    Dp = Dp or (D + 7) // 8 * 8
    hi = torch.empty((M, Dp), dtype=torch.bfloat16, device=x2d.device)
    lo = torch.empty((M, Dp), dtype=torch.bfloat16, device=x2d.device)
    check(lib().ner_split_bf16(ptr(x2d), ptr(hi), ptr(lo), M, D, Dp, x2d.stride(0), stream()))
    return hi, lo


def gemm_split_f32(a_hi, a_lo, w_hi, w_lo, bias=None, residual=None, relu=False, out=None):
    """out f32 [M,N] = [relu](A·W^T + bias [+ residual]) at ~fp32 accuracy: A_hi·W_hi + A_hi·W_lo + A_lo·W_hi
    as three wgmma launches chained through the f32 residual epilogue."""
    M, N = a_hi.shape[0], w_hi.shape[0]
    if out is None:
        out = torch.empty((M, N), dtype=torch.float32, device=a_hi.device)
    gemm_bf16(a_hi, w_hi, bias, residual=residual, epilogue=EPI_RES_F32 if residual is not None else EPI_F32, out=out)
    gemm_bf16(a_hi, w_lo, None, residual=out, epilogue=EPI_RES_F32, out=out)
    gemm_bf16(a_lo, w_hi, None, residual=out, epilogue=EPI_RES_RELU_F32 if relu else EPI_RES_F32, out=out)
    return out


def attention_f32(q, k, v, seq_len, B, L, num_heads, head_dim, scale=1.0, bias_u=None, bias_v=None, rel_table=None,
                  want_f32=True, want_split=False):
    """fp32 attention (+ TENER relative term).  q/k/v: f32 2-D views [B*L, >= heads*head_dim] (row stride = stride(0))."""
    require_cuda(seq_len, bias_u, bias_v, rel_table)
    for t in (q, k, v):
        assert t.is_cuda and t.dtype == torch.float32 and t.dim() == 2 and t.stride(1) == 1 and t.shape[0] == B * L
    HD = num_heads * head_dim
    of = torch.empty((B * L, HD), dtype=torch.float32, device=q.device) if want_f32 else None
    hi = torch.empty((B * L, HD), dtype=torch.bfloat16, device=q.device) if want_split else None
    lo = torch.empty((B * L, HD), dtype=torch.bfloat16, device=q.device) if want_split else None
    check(lib().ner_attention_f32(q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0), v.data_ptr(), v.stride(0),
                                  ptr(bias_u), ptr(bias_v), ptr(rel_table), ptr(_i32(seq_len)), scale, ptr(of), ptr(hi), ptr(lo),
                                  B, L, num_heads, head_dim, stream()))
    return of, hi, lo


def attention_f32_bwd(q, k, v, seq_len, B, L, num_heads, head_dim, d_out, scale=1.0, bias_u=None, bias_v=None, rel_table=None):
    """Backward of attention_f32 -> (dQ, dK, dV [B*L, heads*head_dim] f32, d_bias_u, d_bias_v [heads, head_dim] | None)."""
    require_cuda(seq_len, bias_u, bias_v, rel_table, d_out)
    for t in (q, k, v, d_out):
        assert t.is_cuda and t.dtype == torch.float32 and t.dim() == 2 and t.stride(1) == 1 and t.shape[0] == B * L
    HD = num_heads * head_dim
    dq = torch.empty((B * L, HD), dtype=torch.float32, device=q.device)
    dk = torch.zeros((B * L, HD), dtype=torch.float32, device=q.device)
    dv = torch.zeros((B * L, HD), dtype=torch.float32, device=q.device)
    du = torch.zeros((num_heads, head_dim), dtype=torch.float32, device=q.device) if bias_u is not None else None
    dvb = torch.zeros((num_heads, head_dim), dtype=torch.float32, device=q.device) if bias_v is not None else None
    check(lib().ner_attention_f32_bwd(q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0), v.data_ptr(), v.stride(0),
                                      ptr(bias_u), ptr(bias_v), ptr(rel_table), ptr(_i32(seq_len)), scale, d_out.data_ptr(),
                                      d_out.stride(0), ptr(dq), HD, ptr(dk), HD, ptr(dv), HD, ptr(du), ptr(dvb), B, L, num_heads,
                                      head_dim, stream()))
    return dq, dk, dv, du, dvb


def relu(x, inplace=False):
    require_cuda(x)
    assert x.dtype == torch.float32 and x.is_contiguous()
    y = x if inplace else torch.empty_like(x)
    check(lib().ner_relu_f32(ptr(x), ptr(y), x.numel(), stream()))
    return y


def relu_bwd(act, dact):
    require_cuda(act, dact)
    assert act.dtype == torch.float32 and dact.dtype == torch.float32 and act.numel() == dact.numel()
    out = torch.empty_like(dact)
    check(lib().ner_relu_bwd_f32(ptr(act), ptr(dact), ptr(out), act.numel(), stream()))
    return out


def reduce_max_time(x):
    """tf.reduce_max(x[B,L,C], axis=1) -> [B,C] f32."""
    require_cuda(x)
    assert x.dtype == torch.float32 and x.dim() == 3
    B, L, C = x.shape
    y = torch.empty((B, C), dtype=torch.float32, device=x.device)
    check(lib().ner_reduce_max_time(ptr(x), ptr(y), B, L, C, stream()))
    return y


def reduce_max_time_bwd(x, y, dy, dx, scale=1.0):
    """dx[b,t,c] += scale * dy[b,c] / ties where x == max (TF's reduce_max gradient)."""
    require_cuda(x, y, dy, dx)
    B, L, C = x.shape
    assert dy.dtype == torch.float32 and tuple(dy.shape) == (B, C) and dx.shape == x.shape
    check(lib().ner_reduce_max_time_bwd(ptr(x), ptr(y), ptr(dy), ptr(dx), B, L, C, float(scale), stream()))
    return dx


def softmax_xent(logits, labels, scale=1.0, want_grad=False):
    """sparse softmax cross entropy per row [B, N<=32] -> loss [B] (and scale * (softmax - onehot))."""
    require_cuda(logits, labels)
    assert logits.dtype == torch.float32 and labels.dtype == torch.int32 and logits.dim() == 2
    B, N = logits.shape
    loss = torch.empty((B,), dtype=torch.float32, device=logits.device)
    dz = torch.empty_like(logits) if want_grad else None
    check(lib().ner_softmax_xent(ptr(logits), ptr(labels), ptr(loss), ptr(dz), B, N, float(scale), stream()))
    return (loss, dz) if want_grad else loss


_token_xent_scratch = {}


def _token_head_scratch(dev):
    """The loss-partials buffer of ner_token_xent / ner_token_dice: one per (device, stream)."""
    key = (dev.index, stream())
    scratch = _token_xent_scratch.get(key)
    if scratch is None:
        scratch = _token_xent_scratch[key] = torch.empty(int(lib().ner_token_xent_scratch_floats()), dtype=torch.float32,
                                                         device=dev)
    return scratch


def token_xent(logits, labels=None, seq_len=None, want_pred=True, want_loss=True, want_grad=False, d_loss=1.0):
    """Masked token cross-entropy + first argmax over logits [B, L, K<=32] f32 in one pass (ner_token_xent).
    -> (pred_ids [B,L] int32 | None, loss [] f32 | None, d_logits [B,L,K] | None).  labels None: argmax only.
    loss = mean of (logsumexp - z[label]) over t < seq_len; d_logits = d_loss * its gradient, 0 past seq_len."""
    require_cuda(logits, labels, seq_len)
    assert logits.dtype == torch.float32 and logits.dim() == 3
    B, L, K = logits.shape
    dev = logits.device
    if labels is None:
        want_loss = want_grad = False
    else:
        labels, seq_len = _i32(labels), _i32(seq_len)
        assert tuple(labels.shape) == (B, L) and tuple(seq_len.shape) == (B,)
    pred = torch.empty((B, L), dtype=torch.int32, device=dev) if want_pred else None
    loss = torch.empty((), dtype=torch.float32, device=dev) if want_loss else None
    dz = torch.empty_like(logits) if want_grad else None
    scratch = _token_head_scratch(dev) if labels is not None else None
    check(lib().ner_token_xent(ptr(logits), ptr(labels), ptr(seq_len), ptr(pred), ptr(loss), ptr(dz), float(d_loss),
                               ptr(scratch), B, L, K, stream()))
    if B == 0 and loss is not None:
        loss.zero_()
    if B == 0 and dz is not None:
        dz.zero_()
    return pred, loss, dz


def token_dice(logits, labels, seq_len, alpha=1.0, gamma=1.0, want_pred=True, want_loss=True, want_grad=False, d_loss=1.0):
    """Masked token self-adjusting Dice loss + first argmax over logits [B, L, K<=32] f32 in one pass (ner_token_dice).
    -> (pred_ids [B,L] int32 | None, loss [] f32 | None, d_logits [B,L,K] | None), as token_xent.
    loss = mean over t < seq_len of sum_k dice_k(softmax(z), label; alpha, gamma); d_logits = d_loss * its gradient, 0
    past seq_len.  alpha >= 0, gamma > 0."""
    require_cuda(logits, labels, seq_len)
    assert logits.dtype == torch.float32 and logits.dim() == 3
    B, L, K = logits.shape
    dev = logits.device
    labels, seq_len = _i32(labels), _i32(seq_len)
    assert tuple(labels.shape) == (B, L) and tuple(seq_len.shape) == (B,)
    pred = torch.empty((B, L), dtype=torch.int32, device=dev) if want_pred else None
    loss = torch.empty((), dtype=torch.float32, device=dev) if want_loss else None
    dz = torch.empty_like(logits) if want_grad else None
    check(lib().ner_token_dice(ptr(logits), ptr(labels), ptr(seq_len), ptr(pred), ptr(loss), ptr(dz), float(d_loss),
                               float(alpha), float(gamma), ptr(_token_head_scratch(dev)), B, L, K, stream()))
    if B == 0 and loss is not None:
        loss.zero_()
    if B == 0 and dz is not None:
        dz.zero_()
    return pred, loss, dz


# --------------------------------------------------------------------------- masked-LM pretraining (mlm.py)
def mlm_mask(token_ids, seq_len, pred_offsets, M, seed, V, mask_id, word_start=None):
    """Dynamic whole-word masking (ner_mlm_mask) -> (masked_ids [B,L] i32, positions [M] i32, labels [M] i32).
    pred_offsets [B+1] i32 is the exclusive prefix sum of the per-row budgets and M = pred_offsets[B], known on the host."""
    require_cuda(token_ids, seq_len, pred_offsets, word_start)
    B, L = token_ids.shape
    token_ids, seq_len, pred_offsets = _i32(token_ids), _i32(seq_len), _i32(pred_offsets)
    assert tuple(seq_len.shape) == (B,) and tuple(pred_offsets.shape) == (B + 1,)
    if word_start is not None:
        assert word_start.dtype == torch.uint8 and tuple(word_start.shape) == (B, L)
    dev = token_ids.device
    masked = torch.empty((B, L), dtype=torch.int32, device=dev)
    pos_buf = torch.empty((max(M, 1),), dtype=torch.int32, device=dev)      # one slot at M = 0: never a null pointer
    lab_buf = torch.empty((max(M, 1),), dtype=torch.int32, device=dev)
    check(lib().ner_mlm_mask(ptr(token_ids), ptr(seq_len), ptr(word_start), ptr(pred_offsets), B, L,
                             int(seed) & 0xFFFFFFFFFFFFFFFF, V, mask_id, ptr(masked), ptr(pos_buf), ptr(lab_buf), stream()))
    return masked, pos_buf[:M], lab_buf[:M]


def vocab_xent(logits, labels, V, want_pred=True, want_grad=False, d_loss=1.0):
    """Masked-LM cross-entropy over logits [M, ld] f32, classes in columns < V (ner_vocab_xent).
    -> (loss [] f32, count [] i32, correct [] i32, pred [M] i32 | None, d_logits [M, ld] bf16 | None).  Labels outside
    [0, V) (-1: an unused prediction slot) are not counted; d_logits = d_loss * d loss / d logits, 0 there and in the
    columns >= V."""
    require_cuda(logits, labels)
    assert logits.dtype == torch.float32 and logits.dim() == 2 and labels.dtype == torch.int32
    M, ld = logits.shape
    assert tuple(labels.shape) == (M,)
    dev = logits.device
    loss = torch.zeros((), dtype=torch.float32, device=dev)
    count = torch.zeros((), dtype=torch.int32, device=dev)
    correct = torch.zeros((), dtype=torch.int32, device=dev)
    pred = torch.empty((M,), dtype=torch.int32, device=dev) if want_pred else None
    dz = torch.empty((M, ld), dtype=torch.bfloat16, device=dev) if want_grad else None
    scratch = torch.empty(int(lib().ner_vocab_xent_scratch_floats(M)), dtype=torch.float32, device=dev)
    check(lib().ner_vocab_xent(ptr(logits), ld, ptr(labels), M, V, float(d_loss), ptr(loss), ptr(count), ptr(correct),
                               ptr(pred), ptr(dz), ptr(scratch), stream()))
    return loss, count, correct, pred, dz


# --------------------------------------------------------------------------- training-data augmentation (augment.py)
AUGMENT_MLM_BUDGET = 20        # NER_AUGMENT_MLM_BUDGET


def augment_rows(token_ids, label_ids, seq_len, mask, segment_ids, tables, probs, seed, pad_id, pad_tag, mask_id=-1,
                 want_mlm=False):
    """MR, LwTR, SiS and the masked-LM [MASK]ing of a BIO batch (ner_augment_rows; rules in ner_b200.h).  tables: dict of
    int32 device tensors tag_class [K], type_tag [T,2], mention_type_off [T+1], mention_tok_off [n_mentions+1],
    mention_tokens, tag_tok_off [K+1], tag_tokens (each at least one element).  probs: (row, mr, lwtr, sis, mlm).
    -> dict token_ids, label_ids, mask, segment_ids [B,L], seq_len [B] (i32) and, with want_mlm, mlm_ids [B,L] and
    mlm_positions [B, AUGMENT_MLM_BUDGET]."""
    require_cuda(token_ids, label_ids, seq_len, mask, segment_ids)
    B, L = token_ids.shape
    ids, lab, sl, msk, seg = (_i32(x) for x in (token_ids, label_ids, seq_len, mask, segment_ids))
    tb = tables
    dev = ids.device
    out = {k: torch.empty((B, L), dtype=torch.int32, device=dev) for k in ('token_ids', 'label_ids', 'mask', 'segment_ids')}
    out['seq_len'] = torch.empty((B,), dtype=torch.int32, device=dev)
    if want_mlm:
        out['mlm_ids'] = torch.empty((B, L), dtype=torch.int32, device=dev)
        out['mlm_positions'] = torch.empty((B, AUGMENT_MLM_BUDGET), dtype=torch.int32, device=dev)
    check(lib().ner_augment_rows(
        ptr(ids), ptr(lab), ptr(sl), ptr(msk), ptr(seg), B, L, ptr(tb['tag_class']), tb['tag_class'].numel(),
        ptr(tb['type_tag']), tb['n_types'], ptr(tb['mention_type_off']), ptr(tb['mention_tok_off']),
        ptr(tb['mention_tokens']), tb['n_mentions'], tb['n_mention_tokens'], ptr(tb['tag_tok_off']),
        ptr(tb['tag_tokens']), tb['n_tag_tokens'], *(float(p) for p in probs), int(seed) & 0xFFFFFFFFFFFFFFFF,
        int(pad_id), int(pad_tag), int(mask_id), ptr(out['token_ids']), ptr(out['label_ids']), ptr(out['seq_len']),
        ptr(out['mask']), ptr(out['segment_ids']), ptr(out.get('mlm_ids')), ptr(out.get('mlm_positions')), stream()))
    return out


def vocab_sample(logits, V, eligible, positions, token_ids, temperature, seed):
    """Gumbel-max draw from softmax(logits[:, :V] / temperature) over the eligible ids other than the current one, written
    into token_ids (in place) at positions (ner_vocab_sample; slots at -1 are skipped).  logits [M, ld] f32, eligible [V]
    u8, positions [M] i32."""
    require_cuda(logits, eligible, positions, token_ids)
    assert logits.dtype == torch.float32 and logits.dim() == 2 and eligible.dtype == torch.uint8
    assert positions.dtype == torch.int32 and token_ids.dtype == torch.int32
    M, ld = logits.shape
    assert positions.numel() == M
    check(lib().ner_vocab_sample(ptr(logits), ld, V, ptr(eligible), ptr(positions), M, token_ids.numel(),
                                 float(temperature), int(seed) & 0xFFFFFFFFFFFFFFFF, ptr(token_ids), stream()))
    return token_ids


# --------------------------------------------------------------------------- MRC pairs and tag merge (bert_mrc)
def mrc_pairs(token_ids, seq_len, query_ids, query_len, type_tag, L2, sep_id, label_ids=None):
    """[B, L] BERT batch -> its B*T query/context pairs (ner_mrc_pairs): dict of ids / segment_ids / mask [B*T, L2] i32,
    seq_len [B*T] i32, align [B*T*L] i32 (pair row of each sentence position) and labels [B*T, L] i32 (per-type BIO; None
    without label_ids).  query_ids [T, Qmax] i32, query_len [T] i32, type_tag [T, 2] i32."""
    require_cuda(token_ids, seq_len, query_ids, query_len, type_tag, label_ids)
    B, L = token_ids.shape
    T, Qmax = query_ids.shape
    token_ids, seq_len = _i32(token_ids), _i32(seq_len)
    label_ids = None if label_ids is None else _i32(label_ids)
    assert query_len.dtype == torch.int32 and type_tag.dtype == torch.int32 and tuple(type_tag.shape) == (T, 2)
    dev = token_ids.device
    pair = lambda *shape: torch.empty(shape, dtype=torch.int32, device=dev)
    out = dict(ids=pair(B * T, L2), segment_ids=pair(B * T, L2), mask=pair(B * T, L2), seq_len=pair(B * T),
               align=pair(B * T * L), labels=None if label_ids is None else pair(B * T, L))
    check(lib().ner_mrc_pairs(ptr(token_ids), ptr(seq_len), ptr(label_ids), ptr(query_ids) if Qmax else None, ptr(query_len),
                              ptr(type_tag), B, L, T, Qmax, L2, int(sep_id), ptr(out['ids']), ptr(out['segment_ids']),
                              ptr(out['mask']), ptr(out['seq_len']), ptr(out['labels']), ptr(out['align']), stream()))
    return out


def mrc_merge(logits, seq_len, type_tag, o_id, cls_id, sep_id):
    """Per-type logits [B*T, L, 3] f32 -> pred_ids [B, L] i32 in the dataset's tag space (ner_mrc_merge)."""
    require_cuda(logits, seq_len, type_tag)
    assert logits.dtype == torch.float32 and logits.dim() == 3 and logits.shape[2] == 3
    T = type_tag.shape[0]
    BT, L, _ = logits.shape
    assert BT % T == 0 and type_tag.dtype == torch.int32
    seq_len = _i32(seq_len)
    B = BT // T
    assert tuple(seq_len.shape) == (B,)
    pred = torch.empty((B, L), dtype=torch.int32, device=logits.device)
    check(lib().ner_mrc_merge(ptr(logits), ptr(seq_len), ptr(type_tag), B, L, T, int(o_id), int(cls_id), int(sep_id), ptr(pred),
                              stream()))
    return pred


# --------------------------------------------------------------------------- MRC span pointer (bert_mrc_span)
_span_workspace = {}


def _span_scratch(kind, nbytes, dev):
    """Workspace of one ner_mrc_span_* entry point: one growing buffer per (kind, device, stream)."""
    key = (kind, dev.index, stream())
    buf = _span_workspace.get(key)
    if buf is None or buf.numel() < nbytes:
        buf = _span_workspace[key] = torch.empty(max(int(nbytes), 16), dtype=torch.uint8, device=dev)
    return buf


def _span_uv(uv):
    """[P*L, >= 2I] f32 U | V rows with contiguous rows -> (row stride, I is implied by the caller)."""
    if not uv.is_cuda:
        raise NerB200Error("ner_b200 kernels take CUDA tensors (got a CPU tensor); there is no CPU path")
    assert uv.dtype == torch.float32 and uv.dim() == 2 and uv.stride(1) == 1
    return uv.stride(0)


def mrc_span_targets(pair_labels, pair_seq_len):
    """Per-type BIO labels [P, L] -> (start_y, end_y, span_end) [P, L] i32 (ner_mrc_span_targets)."""
    require_cuda(pair_labels, pair_seq_len)
    P, L = pair_labels.shape
    pair_labels, pair_seq_len = _i32(pair_labels), _i32(pair_seq_len)
    out = [torch.empty((P, L), dtype=torch.int32, device=pair_labels.device) for _ in range(3)]
    check(lib().ner_mrc_span_targets(ptr(pair_labels), ptr(pair_seq_len), P, L, *(ptr(t) for t in out), stream()))
    return tuple(out)


def mrc_span_match_fwd(uv, b1, w2, b2, pair_seq_len, L, span_end=None, keep_prob=1.0, seed=0):
    """Match logits z [P, L, L] f32 (0 off the candidates) and, with span_end, the mean BCE loss [] f32 over the batch's
    candidates (ner_mrc_span_match_fwd).  uv [P*L, >= 2I] f32 (U | V), b1 / w2 [I], b2 [1]."""
    require_cuda(b1, w2, b2, pair_seq_len, span_end)
    ld = _span_uv(uv)
    I = b1.numel()
    P = pair_seq_len.numel()
    dev = uv.device
    z = torch.empty((P, L, L), dtype=torch.float32, device=dev)
    loss = torch.empty((), dtype=torch.float32, device=dev) if span_end is not None else None
    ws, nbytes = None, 0
    if loss is not None:
        nbytes = int(lib().ner_mrc_span_match_fwd_workspace_bytes(P, L))
        ws = _span_scratch('fwd', nbytes, dev)
    check(lib().ner_mrc_span_match_fwd(ptr(uv), ld, ptr(b1), ptr(w2), ptr(b2), ptr(_i32(pair_seq_len)),
                                       ptr(None if span_end is None else _i32(span_end)), P, L, I, float(keep_prob),
                                       int(seed) & 0xFFFFFFFFFFFFFFFF, ptr(z), ptr(loss), ptr(ws), nbytes, stream()))
    if P == 0 and loss is not None:
        loss.zero_()
    return z, loss


def mrc_span_match_bwd(uv, z, b1, w2, pair_seq_len, span_end, d_loss=1.0, keep_prob=1.0, seed=0):
    """-> (d_uv [P*L, 2I], d_b1 [I], d_w2 [I], d_b2 [1]) f32 of d_loss * the forward's loss (ner_mrc_span_match_bwd)."""
    require_cuda(z, b1, w2, pair_seq_len, span_end)
    ld = _span_uv(uv)
    I = b1.numel()
    P, L, _ = z.shape
    dev = uv.device
    d_uv = torch.empty((P * L, 2 * I), dtype=torch.float32, device=dev)
    d_b1 = torch.empty((I,), dtype=torch.float32, device=dev)
    d_w2 = torch.empty((I,), dtype=torch.float32, device=dev)
    d_b2 = torch.empty((1,), dtype=torch.float32, device=dev)
    nbytes = int(lib().ner_mrc_span_match_bwd_workspace_bytes(P, I))
    ws = _span_scratch('bwd', nbytes, dev)
    check(lib().ner_mrc_span_match_bwd(ptr(uv), ld, ptr(z), ptr(b1), ptr(w2), ptr(_i32(pair_seq_len)), ptr(_i32(span_end)), P, L,
                                       I, float(d_loss), float(keep_prob), int(seed) & 0xFFFFFFFFFFFFFFFF, ptr(d_uv), ptr(d_b1),
                                       ptr(d_w2), ptr(d_b2), ptr(ws), nbytes, stream()))
    if P == 0:
        for t in (d_uv, d_b1, d_w2, d_b2):
            t.zero_()
    return d_uv, d_b1, d_w2, d_b2


def mrc_span_decode(start_logits, end_logits, uv, b1, w2, b2, seq_len, type_tag, o_id, cls_id, sep_id, cap=None):
    """Start / end logits [B*T, L, 2] f32 and U | V rows -> pred_ids [B, L] i32 carrying .spans [B, cap] i32,
    .span_probs [B, cap] f32 and .span_counts [B] i32 (ner_mrc_span_decode).  cap None = L."""
    require_cuda(start_logits, end_logits, b1, w2, b2, seq_len, type_tag)
    assert start_logits.dtype == torch.float32 and end_logits.dtype == torch.float32
    ld = _span_uv(uv)
    T = type_tag.shape[0]
    P, L, _ = start_logits.shape
    B = P // T
    I = b1.numel()
    cap = L if cap is None else int(cap)
    dev = start_logits.device
    pred = torch.empty((B, L), dtype=torch.int32, device=dev)
    spans = torch.empty((B, cap), dtype=torch.int32, device=dev)
    probs = torch.empty((B, cap), dtype=torch.float32, device=dev)
    counts = torch.empty((B,), dtype=torch.int32, device=dev)
    nbytes = int(lib().ner_mrc_span_decode_workspace_bytes(P, L))
    ws = _span_scratch('decode', nbytes, dev)
    check(lib().ner_mrc_span_decode(ptr(start_logits.contiguous()), ptr(end_logits.contiguous()), ptr(uv), ld, ptr(b1), ptr(w2),
                                    ptr(b2), ptr(_i32(seq_len)), ptr(type_tag), B, T, L, I, int(o_id), int(cls_id), int(sep_id),
                                    cap, ptr(pred), ptr(spans), ptr(probs), ptr(counts), ptr(ws), nbytes, stream()))
    if B == 0:
        counts.zero_()
    pred.spans, pred.span_probs, pred.span_counts = spans, probs, counts
    return pred


# --------------------------------------------------------------------------- GlobalPointer span head (bert_global_pointer)
GP_HEAD = 64                                     # D, the head size of ner_gp_*


def _gp_rows(rot, B, L, cu_seqlens):
    """rot [rows, T, 2, D] bf16 -> T; rows must be B*L (padded) or the packed count (checked by the caller's layout)."""
    require_cuda(rot, cu_seqlens)
    assert rot.dtype == torch.bfloat16 and rot.dim() == 4 and rot.shape[2] == 2 and rot.shape[3] == GP_HEAD
    assert cu_seqlens is not None or rot.shape[0] == B * L
    return rot.shape[1]


def gp_targets(label_ids, seq_len, type_tag):
    """label_ids [B, L] -> span_end [B, T, L] i32 (ner_gp_targets)."""
    require_cuda(label_ids, seq_len, type_tag)
    B, L = label_ids.shape
    T = type_tag.shape[0]
    assert type_tag.dtype == torch.int32 and tuple(type_tag.shape) == (T, 2)
    out = torch.empty((B, T, L), dtype=torch.int32, device=label_ids.device)
    check(lib().ner_gp_targets(ptr(_i32(label_ids)), ptr(_i32(seq_len)), ptr(type_tag), B, T, L, ptr(out), stream()))
    return out


def gp_rope(proj, B, L, T, cu_seqlens=None, split=False):
    """proj [rows, >= T*2D] f32 (q | k of each type) -> (hi, lo | None) bf16 [rows, T, 2, D]: the rotated operands, q
    scaled by 1/sqrt(D) (ner_gp_rope).  split: lo = the bf16 rest of the fp32 value."""
    _require_rows(proj)
    require_cuda(cu_seqlens)
    rows = proj.shape[0]
    hi = torch.empty((rows, T, 2, GP_HEAD), dtype=torch.bfloat16, device=proj.device)
    lo = torch.empty_like(hi) if split else None
    check(lib().ner_gp_rope(ptr(proj), proj.stride(0), ptr(cu_seqlens), B, T, L, ptr(hi), ptr(lo), stream()))
    return hi, lo


def gp_rope_bwd(d_rot, B, L, cu_seqlens=None):
    """d_rot [rows, T, 2, D] f32 -> d_proj [rows, T*2D] f32 (ner_gp_rope_bwd)."""
    require_cuda(d_rot, cu_seqlens)
    rows, T = d_rot.shape[:2]
    d_proj = torch.empty((rows, T * 2 * GP_HEAD), dtype=torch.float32, device=d_rot.device)
    check(lib().ner_gp_rope_bwd(ptr(d_rot), ptr(cu_seqlens), B, T, L, ptr(d_proj), d_proj.stride(0), stream()))
    return d_proj


def gp_loss_fwd(hi, lo, seq_len, span_end, L, cu_seqlens=None):
    """-> (loss [] f32, lse [B, T, 2] f32) of the multilabel span cross-entropy (ner_gp_loss_fwd); lo None = bf16 scores."""
    require_cuda(lo, seq_len, span_end)
    B = seq_len.shape[0]
    T = _gp_rows(hi, B, L, cu_seqlens)
    assert tuple(span_end.shape) == (B, T, L) and span_end.dtype == torch.int32
    dev = hi.device
    loss = torch.zeros((), dtype=torch.float32, device=dev)
    lse = torch.zeros((B, T, 2), dtype=torch.float32, device=dev)
    nbytes = int(lib().ner_gp_loss_workspace_bytes(B, T, L))
    ws = _span_scratch('gp_loss', nbytes, dev)
    check(lib().ner_gp_loss_fwd(ptr(hi), ptr(lo), ptr(_i32(seq_len)), ptr(cu_seqlens), ptr(span_end), B, T, L, ptr(loss),
                                ptr(lse), ptr(ws), nbytes, stream()))
    return loss, lse


def gp_loss_bwd(rot, seq_len, span_end, lse, L, d_loss=1.0, cu_seqlens=None):
    """-> d_rot [rows, T, 2, D] f32, the gradient of d_loss * the loss w.r.t. the rotated operands (ner_gp_loss_bwd)."""
    require_cuda(seq_len, span_end, lse)
    B = seq_len.shape[0]
    T = _gp_rows(rot, B, L, cu_seqlens)
    d_rot = torch.zeros(rot.shape, dtype=torch.float32, device=rot.device)
    check(lib().ner_gp_loss_bwd(ptr(rot), ptr(_i32(seq_len)), ptr(cu_seqlens), ptr(span_end), ptr(lse), B, T, L,
                                float(d_loss), ptr(d_rot), stream()))
    return d_rot


def gp_decode(hi, lo, seq_len, type_tag, o_id, cls_id, sep_id, L, cu_seqlens=None, cap=None, want_scores=False):
    """Rotated operands -> pred_ids [B, L] i32 carrying .spans [B, cap] i32, .span_probs [B, cap] f32 and .span_counts [B]
    i32 (ner_gp_decode).  cap None = L.  want_scores: also return the scores [B, T, L, L] f32 (valid at the candidates
    only; a view of the workspace, overwritten by the next call on this stream)."""
    require_cuda(lo, seq_len, type_tag)
    B = seq_len.shape[0]
    T = _gp_rows(hi, B, L, cu_seqlens)
    assert tuple(type_tag.shape) == (T, 2) and type_tag.dtype == torch.int32
    cap = L if cap is None else int(cap)
    dev = hi.device
    pred = torch.empty((B, L), dtype=torch.int32, device=dev)
    spans = torch.empty((B, cap), dtype=torch.int32, device=dev)
    probs = torch.empty((B, cap), dtype=torch.float32, device=dev)
    counts = torch.zeros((B,), dtype=torch.int32, device=dev)
    nbytes = int(lib().ner_gp_decode_workspace_bytes(B, T, L))
    ws = _span_scratch('gp_decode', nbytes, dev)
    check(lib().ner_gp_decode(ptr(hi), ptr(lo), ptr(_i32(seq_len)), ptr(cu_seqlens), ptr(type_tag), B, T, L, int(o_id),
                              int(cls_id), int(sep_id), cap, ptr(pred), ptr(spans), ptr(probs), ptr(counts), ptr(ws), nbytes,
                              stream()))
    pred.spans, pred.span_probs, pred.span_counts = spans, probs, counts
    if want_scores:
        return pred, ws[:nbytes].view(torch.float32).view(B, T, L, L)
    return pred


# --------------------------------------------------------------------------- document windows (BERT document mode)
def window_plan(token_ids, segment_ids, seq_len, W, S, NW, n_doc, packed=False, padded=False):
    """[B, L] documents -> their W-token windows (ner_window_plan): dict of ids / segment_ids / mask [NW, W] i32 and the
    owner row of every document token (n_doc of them, documents back to back) in the window-packed layout
    (doc_src_packed, when packed) and the window-padded one (doc_src_padded, when padded).  NW and n_doc are host counts
    (windows.window_counts and the mask's token count)."""
    require_cuda(token_ids, segment_ids, seq_len)
    B, L = token_ids.shape
    token_ids, seq_len = _i32(token_ids), _i32(seq_len)
    segment_ids = None if segment_ids is None else _i32(segment_ids)
    dev = token_ids.device
    i32 = lambda *shape: torch.empty(shape, dtype=torch.int32, device=dev)
    out = dict(ids=i32(NW, W), segment_ids=i32(NW, W), mask=i32(NW, W), doc_src_packed=i32(n_doc) if packed else None,
               doc_src_padded=i32(n_doc) if padded else None)
    check(lib().ner_window_plan(ptr(token_ids), ptr(segment_ids), ptr(seq_len), B, L, int(W), int(S), int(NW), ptr(out['ids']),
                                ptr(out['segment_ids']), ptr(out['mask']), ptr(out['doc_src_packed']),
                                ptr(out['doc_src_padded']), stream()))
    return out


# --------------------------------------------------------------------------- training-side kernels
def _require_rows(x2d):
    """CUDA f32 2-D tensor whose rows are contiguous (a column slice of a wider buffer is fine)."""
    if not x2d.is_cuda:
        raise _lib.NerB200Error("ner_b200 kernels take CUDA tensors (got a CPU tensor); there is no CPU path")
    assert x2d.dtype == torch.float32 and x2d.dim() == 2 and x2d.stride(1) == 1


def transpose_cast_bf16(x2d, Mp=None):
    """f32 [M,N] -> bf16 [N,Mp]: K-major operand of a weight-gradient GEMM (reduction over the M rows)."""
    _require_rows(x2d)
    M, N = x2d.shape
    Mp = Mp or (M + 7) // 8 * 8
    out = torch.empty((N, Mp), dtype=torch.bfloat16, device=x2d.device)
    check(lib().ner_transpose_cast_bf16(ptr(x2d), ptr(out), M, N, Mp, x2d.stride(0), stream()))
    return out


def wgrad_gemm(x2d, dy2d, out=None):
    """dW [K,N] f32 = x^T [K,M] · dy [M,N] on the tensor cores (bf16 operands, fp32 accumulate)."""
    M = x2d.shape[0]
    Mp = (M + 7) // 8 * 8
    xt = transpose_cast_bf16(x2d, Mp)        # [K, Mp]
    dyt = transpose_cast_bf16(dy2d, Mp)      # [N, Mp]
    N = dyt.shape[0]
    if N % 32 != 0:                          # pad the output columns to the GEMM's 32-column granule
        Np = (N + 31) // 32 * 32
        dyt = torch.nn.functional.pad(dyt, (0, 0, 0, Np - N))
    res = gemm_bf16(xt, dyt.contiguous(), None, epilogue=EPI_F32)
    res = res[:, :N] if res.shape[1] != N else res
    if out is not None:
        out.add_(res)
        return out
    return res.contiguous()


def colsum_add(x2d, out, scale=1.0):
    _require_rows(x2d)
    require_cuda(out)
    M, N = x2d.shape
    check(lib().ner_colsum_add(ptr(x2d), ptr(out), M, N, x2d.stride(0), scale, stream()))
    return out


def dense_small_n_bwd(x2d, w, dy, dW, db=None, want_dx=True):
    require_cuda(x2d, w, dy, dW, db)
    assert x2d.dtype == torch.float32
    M, F = x2d.shape
    N = w.shape[1]
    dx = torch.empty((M, F), dtype=torch.float32, device=x2d.device) if want_dx else None
    check(lib().ner_dense_small_n_bwd(ptr(x2d), ptr(w), ptr(dy), ptr(dW), ptr(db), ptr(dx), M, F, N, stream()))
    return dx


def dropout(x, keep_prob, seed, inplace=False):
    """tf.layers.dropout forward (and backward: same call on the gradient with the same seed); f32 or bf16."""
    require_cuda(x)
    assert x.dtype in (torch.float32, torch.bfloat16) and x.is_contiguous()
    y = x if inplace else torch.empty_like(x)
    fn = lib().ner_dropout if x.dtype == torch.float32 else lib().ner_dropout_bf16
    check(fn(ptr(x), ptr(y), x.numel(), float(keep_prob), int(seed) & 0xFFFFFFFFFFFFFFFF, stream()))
    return y


_sumsq_scratch = {}


def sumsq_add(g, out):
    require_cuda(g, out)
    key = (g.device.index, stream())
    scratch = _sumsq_scratch.get(key)
    if scratch is None:
        scratch = _sumsq_scratch[key] = torch.empty(int(lib().ner_sumsq_scratch_floats()), dtype=torch.float32, device=g.device)
    check(lib().ner_sumsq_add(ptr(g), g.numel(), ptr(out), ptr(scratch), stream()))
    return out


def adam_step(p, g, m, v, lr, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.0, mode=1, clip=0.0, gnorm_sq=None,
              grad_scale=1.0):
    """mode 0: AdamWeightDecayOptimizer (bert), mode 1: tf.train.AdamOptimizer; flat f32 buffers."""
    require_cuda(p, g, m, v, gnorm_sq)
    n = p.numel()
    assert g.numel() == n and m.numel() == n and v.numel() == n
    check(lib().ner_adam_step(ptr(p), ptr(g), ptr(m), ptr(v), n, lr, beta1, beta2, eps, weight_decay, mode, clip,
                              ptr(gnorm_sq), grad_scale, stream()))


# --------------------------------------------------------------------------- encoder backward
def layernorm_bwd(y, gamma, d_out, d_gamma, d_beta, residual=None, eps=1e-12, want_f32=True, want_bf16=True, keep_prob=1.0,
                  seed=0, d_bias=None):
    """d_bias (optional, [H] f32, accumulated into): column sums of the masked dense-branch gradient = the bias gradient of
    the dense layer whose output this LayerNorm normalises."""
    require_cuda(y, gamma, d_out, d_gamma, d_beta, residual, d_bias)
    M, H = y.shape
    dz32 = torch.empty((M, H), dtype=torch.float32, device=y.device) if want_f32 else None
    dz16 = torch.empty((M, H), dtype=torch.bfloat16, device=y.device) if want_bf16 else None
    check(lib().ner_layernorm_dropout_bwd_bias(ptr(y), 1 if y.dtype == torch.bfloat16 else 0, ptr(residual), ptr(gamma),
                                               ptr(d_out), ptr(dz32), ptr(dz16), ptr(d_gamma), ptr(d_beta), ptr(d_bias), M, H, eps,
                                               float(keep_prob), int(seed) & 0xFFFFFFFFFFFFFFFF, stream()))
    return dz32, dz16


def transpose_bf16(x, Mp=None):
    require_cuda(x)
    assert x.dtype == torch.bfloat16 and x.dim() == 2
    M, N = x.shape
    Mp = Mp or (M + 7) // 8 * 8
    out = torch.empty((N, Mp), dtype=torch.bfloat16, device=x.device)
    check(lib().ner_transpose_bf16(ptr(x), ptr(out), M, N, Mp, stream()))
    return out


def wgrad_gemm_bf16(x16, dy16, out_f32=None):
    """dW [K,N] f32 (+)= x^T · dy for bf16 activations x [M,K], dy [M,N] (tensor cores, fp32 accumulate)."""
    M = x16.shape[0]
    Mp = (M + 7) // 8 * 8
    xt, dyt = transpose_bf16(x16, Mp), transpose_bf16(dy16, Mp)
    if out_f32 is None:
        return gemm_bf16(xt, dyt, None, epilogue=EPI_F32)
    return gemm_bf16(xt, dyt, None, residual=out_f32, epilogue=EPI_RES_F32, out=out_f32)


def colsum_bf16_add(x16, out):
    require_cuda(x16, out)
    M, N = x16.shape
    check(lib().ner_colsum_bf16_add(ptr(x16), ptr(out), M, N, stream()))
    return out


def gelu_bf16(pre, erf=False):
    require_cuda(pre)
    out = torch.empty_like(pre)
    check(lib().ner_gelu_bf16(ptr(pre), ptr(out), pre.numel(), 1 if erf else 0, stream()))
    return out


def gelu_f32(x, erf=False, inplace=False):
    require_cuda(x)
    assert x.dtype == torch.float32 and x.is_contiguous()
    y = x if inplace else torch.empty_like(x)
    check(lib().ner_gelu_f32(ptr(x), ptr(y), x.numel(), 1 if erf else 0, stream()))
    return y


def gelu_bwd_bias_bf16(pre, dact, d_bias, erf=False):
    """d_pre = d_act * gelu'(pre) and d_bias += column sums of d_pre, one pass (pre / dact bf16 [M, N])."""
    require_cuda(pre, dact, d_bias)
    M, N = pre.shape
    out = torch.empty_like(pre)
    check(lib().ner_gelu_bwd_bias_bf16(ptr(pre), ptr(dact), ptr(out), ptr(d_bias), M, N, 1 if erf else 0, stream()))
    return out


def gelu_bwd_bf16(pre, dact, erf=False):
    require_cuda(pre, dact)
    out = torch.empty_like(pre)
    check(lib().ner_gelu_bwd_bf16(ptr(pre), ptr(dact), ptr(out), pre.numel(), 1 if erf else 0, stream()))
    return out


def bert_embed_bwd(dx, ids, seg, d_word, d_type, d_pos):
    require_cuda(dx, ids, seg, d_word, d_type, d_pos)
    B, L = ids.shape
    H = dx.shape[-1]
    check(lib().ner_bert_embed_bwd(ptr(dx), ptr(_i32(ids)), ptr(None if seg is None else _i32(seg)), ptr(d_word), ptr(d_type),
                                   ptr(d_pos), B, L, H, d_word.shape[0], d_type.shape[0], stream()))


def gather_rows(src2d, idx, n):
    """dst row r = src row idx[r] for r < n (padded -> packed layout)."""
    require_cuda(src2d, idx)
    assert idx.dtype == torch.int32 and src2d.dim() == 2
    dst = torch.empty((n, src2d.shape[1]), dtype=src2d.dtype, device=src2d.device)
    check(lib().ner_gather_rows(ptr(src2d), ptr(idx), ptr(dst), n, src2d.shape[1] * src2d.element_size(), stream()))
    return dst


def scatter_rows(src2d, idx, rows):
    """dst [rows, C] zeros with dst row idx[r] = src row r (packed -> padded layout)."""
    require_cuda(src2d, idx)
    assert idx.dtype == torch.int32 and src2d.dim() == 2
    dst = torch.zeros((rows, src2d.shape[1]), dtype=src2d.dtype, device=src2d.device)
    check(lib().ner_scatter_rows(ptr(src2d), ptr(idx), ptr(dst), src2d.shape[0], src2d.shape[1] * src2d.element_size(), stream()))
    return dst


def bert_attention_bwd(qkv, mask, ctx, dctx, B, L, num_heads, head_dim=64, scale=None, mask_add=-10000.0, keep_prob=1.0, seed=0,
                       cu_seqlens=None):
    require_cuda(qkv, mask, ctx, dctx, cu_seqlens)
    assert qkv.dtype == torch.bfloat16 and ctx.dtype == torch.bfloat16 and dctx.dtype == torch.bfloat16
    dqkv = torch.empty_like(qkv)
    if scale is None:
        scale = 1.0 / (head_dim ** 0.5)
    if cu_seqlens is not None:
        check(lib().ner_bert_attention_bwd_packed(ptr(qkv), ptr(cu_seqlens), ptr(ctx), ptr(dctx), ptr(dqkv), B, L, num_heads, head_dim,
                                                  scale, float(keep_prob), int(seed) & 0xFFFFFFFFFFFFFFFF, stream()))
        return dqkv
    check(lib().ner_bert_attention_bwd(ptr(qkv), ptr(_i32(mask)), ptr(ctx), ptr(dctx), ptr(dqkv), B, L, num_heads, head_dim,
                                       scale, mask_add, float(keep_prob), int(seed) & 0xFFFFFFFFFFFFFFFF, stream()))
    return dqkv


# --------------------------------------------------------------------------- entity spans (serving tail)
def tag_classes(idx2tag):
    """idx2tag -> (class table [K] for ner_extract_spans, list of entity types).  The table is uint8 (5 type bits) up to
    32 entity types, and int16 for ner_extract_spans_wide (7 type bits) up to 128."""
    K = max(idx2tag) + 1
    types, table = [], [0] * K
    for i, tag in idx2tag.items():
        head = tag.split('-')[0]
        kind = 1 if head == 'B' else 2 if head == 'I' else 0
        t = 0
        if kind and '-' in tag:
            name = tag.split('-')[1]
            if name not in types:
                types.append(name)
            t = types.index(name)
        table[i] = kind | (4 if tag[:1] in ('B', 'I') else 0) | (t << 3)
    assert len(types) <= 128
    return torch.tensor(table, dtype=torch.uint8 if len(types) <= 32 else torch.int16), types


def extract_spans(pred_ids, tag_class, cap=None):
    """pred_ids [B,L] int32 (device), tag_class uint8 [K] (device) -> (spans int32 [B,cap], counts int32 [B])."""
    require_cuda(pred_ids, tag_class)
    B, L = pred_ids.shape
    cap = cap or L            # 'B B B ...': every position can be a span of its own
    spans = torch.empty((B, cap), dtype=torch.int32, device=pred_ids.device)
    counts = torch.empty((B,), dtype=torch.int32, device=pred_ids.device)
    fn = lib().ner_extract_spans if tag_class.dtype == torch.uint8 else lib().ner_extract_spans_wide
    assert tag_class.dtype in (torch.uint8, torch.int16)
    check(fn(ptr(_i32(pred_ids)), ptr(tag_class), ptr(spans), ptr(counts), B, L, tag_class.numel(), cap, stream()))
    return spans, counts


# --------------------------------------------------------------------------- raw text -> features (serving head)
def _featurize_args(text_dev, offsets_host, B, uni, vocab, out):
    require_cuda(text_dev, *out.values())
    head = 8 * (B + 1)
    return ([ptr(text_dev) + head, ptr(text_dev), offsets_host.data_ptr(), B],
            [vocab['slots'].data_ptr(), vocab['slots'].numel(), ptr(vocab['entries']), ptr(vocab['blob'])],
            [ptr(out[k]) for k in ('token_ids', 'mask', 'segment_ids', 'seq_len', 'unk_cursor')] + [stream()])


def featurize_wordpiece(text_dev, offsets_host, B, L, uni, vocab, max_piece, lower, special, out):
    """ner_featurize_wordpiece.  text_dev uint8 (device) = offsets int64 [B+1] then the UTF-8 bytes; offsets_host the
    host buffer it was copied from; uni / vocab the device tables of data/device_featurize.py; special = ([CLS], [SEP],
    [PAD], [UNK]) ids; out the five [B, L] / [B] int32 outputs."""
    head, tab, tail = _featurize_args(text_dev, offsets_host, B, uni, vocab, out)
    check(lib().ner_featurize_wordpiece(*head, L, ptr(uni['stage1']), ptr(uni['stage2']), ptr(uni['expand']), *tab,
                                        int(max_piece), int(bool(lower)), *special, *tail))


def featurize_chars(text_dev, offsets_host, B, L, uni, vocab, max_piece, lower, special, out):
    """ner_featurize_chars: as featurize_wordpiece with special = ([PAD], [UNK]) ids (max_piece / lower unused)."""
    head, tab, tail = _featurize_args(text_dev, offsets_host, B, uni, vocab, out)
    check(lib().ner_featurize_chars(*head, L, ptr(uni['stage1']), ptr(uni['stage2']), *tab, *special, *tail))


def wgrad_group(problems, rows):
    """problems: list of (x bf16 [rows, ld_x], dy bf16 [rows, ld_dy], dy_col0, dw f32 [k_in, n_out]) -> dw += x[:, :k_in]^T dy[:, col0:col0+n_out],
    all in one launch (ner_wgrad_group_bf16)."""
    from ._lib import WgradProblem
    arr = (WgradProblem * len(problems))()
    for q, (x, dy, col0, dw) in zip(arr, problems):
        require_cuda(x, dy, dw)
        assert x.dtype == torch.bfloat16 and dy.dtype == torch.bfloat16 and dw.dtype == torch.float32
        q.x_bf16, q.ld_x, q.dy_bf16, q.ld_dy, q.dy_col0 = ptr(x), x.shape[1], ptr(dy), dy.shape[1], int(col0)
        q.dw, q.k_in, q.n_out = ptr(dw), dw.shape[0], dw.shape[1]
    check(lib().ner_wgrad_group_bf16(arr, len(problems), int(rows), stream()))


class PackGroup(object):
    """A fixed set of (f32 kernel [K,N], bf16 [N,K] pack view, bf16 [K,N] cast view) triples re-packed by ONE launch
    (ner_pack_weights_group_bf16).  The table lives on the device; `run()` after every optimizer step."""

    def __init__(self, triples):
        import ctypes
        from ._lib import PackEntry
        arr = (PackEntry * len(triples))()
        starts = [0]
        self.keep = triples
        for q, (src, nk, kn) in zip(arr, triples):
            require_cuda(src)
            for t in (nk, kn):          # destinations may be row / column blocks of a fused operand: unit stride along the row only
                if t is not None and not (t.is_cuda and t.dtype == torch.bfloat16 and t.stride(1) == 1):
                    raise NerB200Error("PackGroup destinations must be CUDA bf16 matrices with contiguous rows")
            K, N = src.shape
            assert src.dtype == torch.float32 and src.is_contiguous()
            q.src, q.K, q.N = ptr(src), K, N
            q.dst_nk_bf16, q.ld_nk = (ptr(nk), nk.stride(0)) if nk is not None else (0, 0)
            q.dst_kn_bf16, q.ld_kn = (ptr(kn), kn.stride(0)) if kn is not None else (0, 0)
            starts.append(starts[-1] + ((K + 63) // 64) * ((N + 63) // 64))
        dev = triples[0][0].device
        raw = bytes(memoryview(arr))
        self.table = torch.frombuffer(bytearray(raw), dtype=torch.uint8).to(dev)
        self.starts = torch.tensor(starts, dtype=torch.int32, device=dev)
        self.count, self.tiles = len(triples), starts[-1]
        self.signature = tuple(ptr(t[0]) for t in triples)

    def run(self):
        check(lib().ner_pack_weights_group_bf16(ptr(self.table), ptr(self.starts), self.count, self.tiles, stream()))
