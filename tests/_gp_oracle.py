"""float64 restatement of the GlobalPointer head of bert_global_pointer (include/ner_b200.h: ner_gp_targets, ner_gp_rope,
ner_gp_loss_fwd / _bwd, ner_gp_decode): projection, RoPE, scores, targets, the multilabel span cross-entropy and its dS,
and the decode.  Projection, RoPE, scores and loss are torch (differentiable, on whatever device their inputs are on);
targets and decode are numpy, the greedy projection is _mrc_span_oracle's."""
import numpy as np
import torch

from _mrc_span_oracle import project, sigmoid32

D = 64


def projection(h, kernel, bias, T):
    """h [..., H] @ kernel [H, T*2D] + bias -> (q, k) [..., T, D] (bert4keras layout: q of type t, then its k)."""
    P = h @ kernel + bias
    P = P.reshape(*P.shape[:-1], T, 2, D)
    return P[..., 0, :], P[..., 1, :]


def rope(x, pos):
    """x [B, L, ..., D] rotated pair (2i, 2i+1) by pos[s] * 10000^(-2i/D) at sentence position s."""
    i = torch.arange(D // 2, dtype=torch.float64, device=x.device)
    theta = 10000.0 ** (-2.0 * i / D)
    pos = torch.as_tensor(pos, dtype=torch.float64, device=x.device)
    ang = pos[:, None] * theta[None, :]                                     # [L, D/2]
    shape = [1, len(pos)] + [1] * (x.dim() - 3) + [D // 2]
    c, s = torch.cos(ang).view(shape).to(x.dtype), torch.sin(ang).view(shape).to(x.dtype)
    x0, x1 = x[..., 0::2], x[..., 1::2]
    return torch.stack([x0 * c - x1 * s, x1 * c + x0 * s], dim=-1).flatten(-2)


def operands(q, k):
    """q, k [B, L, T, D] -> q' = RoPE(q) / sqrt(D), k' = RoPE(k) (position = index in the padded sentence)."""
    pos = np.arange(q.shape[1])
    return rope(q, pos) / np.sqrt(D), rope(k, pos)


def scores(qr, kr):
    """q', k' [B, L, T, D] -> s [B, T, L, L] = q'_i . k'_j."""
    return torch.einsum('bitd,bjtd->btij', qr, kr)


def targets(label_ids, seq_len, type_tag):
    """label_ids [B, L], type_tag [T, 2] (B-X, I-X ids) -> span_end [B, T, L] int32."""
    label_ids = np.asarray(label_ids)
    B, L = label_ids.shape
    T = len(type_tag)
    out = np.full((B, T, L), -1, np.int32)
    for b in range(B):
        n = min(max(int(seq_len[b]), 0), L)
        y = label_ids[b, :n]
        for t, (tb, ti) in enumerate(type_tag):
            for s in range(n):
                if y[s] == tb:
                    r = s
                    while r + 1 < n and y[r + 1] == ti:
                        r += 1
                    out[b, t, s] = r
    return out


def candidates(seq_len, L):
    """[B, L, L] bool: 1 <= i <= j <= len - 2."""
    i = np.arange(L)[:, None]
    j = np.arange(L)[None, :]
    out = np.zeros((len(seq_len), L, L), bool)
    for b, n in enumerate(seq_len):
        m = min(max(int(n), 0), L) - 2
        out[b] = (i >= 1) & (i <= j) & (j <= m)
    return out


def _sets(S, span_end, seq_len):
    B, T, L, _ = S.shape
    cand = torch.as_tensor(candidates(seq_len, L), device=S.device)[:, None]            # [B, 1, L, L]
    pos = torch.as_tensor(np.asarray(span_end)[..., None] == np.arange(L), device=S.device) & cand
    return cand & ~pos, pos


def lse(S, span_end, seq_len):
    """-> (lse_neg, lse_pos) [B, T]: log(1 + sum_neg e^s), log(1 + sum_pos e^-s)."""
    neg, pos = _sets(S, span_end, seq_len)
    ninf = torch.tensor(-np.inf, dtype=S.dtype, device=S.device)
    zero = torch.zeros(S.shape[:2] + (1,), dtype=S.dtype, device=S.device)
    ln = torch.logsumexp(torch.cat([zero, torch.where(neg, S, ninf).flatten(2)], -1), -1)
    lp = torch.logsumexp(torch.cat([zero, torch.where(pos, -S, ninf).flatten(2)], -1), -1)
    return ln, lp


def loss(S, span_end, seq_len):
    """Mean over B*T of lse_neg + lse_pos (differentiable)."""
    ln, lp = lse(S, span_end, seq_len)
    return (ln + lp).mean()


def d_scores(S, span_end, seq_len, d_loss=1.0):
    """dS of d_loss * loss: e^(s - lse_neg) on negatives, -e^(-s - lse_pos) on positives, 0 elsewhere, / (B*T)."""
    neg, pos = _sets(S, span_end, seq_len)
    ln, lp = lse(S, span_end, seq_len)
    g = d_loss / (S.shape[0] * S.shape[1])
    out = torch.where(neg, torch.exp(S - ln[..., None, None]), torch.zeros_like(S))
    return g * torch.where(pos, -torch.exp(-S - lp[..., None, None]), out)


def decode(S, seq_len, type_tag, o_id, cls_id, sep_id, cap):
    """s [B, T, L, L] f32 (read at the candidates only) -> (pred_ids [B, L], spans [B, cap], probs [B, cap], counts [B]);
    entries past the count are 0."""
    S = np.asarray(S, np.float32)
    B, T, L, _ = S.shape
    pred = np.zeros((B, L), np.int32)
    words = np.zeros((B, cap), np.int32)
    probs = np.zeros((B, cap), np.float32)
    counts = np.zeros(B, np.int32)
    for b in range(B):
        n = min(max(int(seq_len[b]), 0), L)
        m = n - 2
        spans = [(i, j, t, float(S[b, t, i, j])) for i in range(1, m + 1) for j in range(i, m + 1) for t in range(T)
                 if S[b, t, i, j] > 0]
        counts[b] = len(spans)
        for o, (i, j, t, zz) in enumerate(spans[:cap]):
            words[b, o] = i | (j + 1) << 12 | t << 24
            probs[b, o] = sigmoid32(zz)
        pred[b] = project(spans, n, type_tag, o_id, cls_id, sep_id, L)
    return pred, words, probs, counts
