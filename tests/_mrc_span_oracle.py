"""float64 restatement of the bert_mrc_span head (include/ner_b200.h: ner_mrc_span_targets, ner_mrc_span_match_fwd /
_bwd, ner_mrc_span_decode): the targets, the dropout hash, the match logits, the BCE loss over the candidates, the decode
and the greedy projection.  The match head runs in torch float64 (differentiable, on whatever device its inputs are on) so
the GPU tests can restate full-size problems pair by pair; everything else is numpy."""
import numpy as np
import torch

C0 = np.sqrt(2.0 / np.pi)
M32 = 0xFFFFFFFF


def targets(labels, seq_len):
    """Per-type BIO labels [P, L] (0 O, 1 B, 2 I) -> (start_y, end_y, span_end) [P, L] int32."""
    labels = np.asarray(labels)
    P, L = labels.shape
    start = np.zeros((P, L), np.int32)
    end = np.zeros((P, L), np.int32)
    span_end = np.full((P, L), -1, np.int32)
    for p in range(P):
        n = min(max(int(seq_len[p]), 0), L)
        y = labels[p, :n]
        for s in range(n):
            if y[s] == 1:
                r = s
                while r + 1 < n and y[r + 1] == 2:
                    r += 1
                start[p, s] = 1
                span_end[p, s] = r
                end[p, r] = 1
    return start, end, span_end


def candidates(seq_len, L):
    """[P, L, L] bool: 1 <= i <= j <= len - 2."""
    P = len(seq_len)
    i = np.arange(L)[:, None]
    j = np.arange(L)[None, :]
    out = np.zeros((P, L, L), bool)
    for p in range(P):
        m = min(max(int(seq_len[p]), 0), L) - 2
        out[p] = (i >= 1) & (i <= j) & (j <= m)
    return out


def _hash3(a, b, c):
    """nerdev::hash3 on int64 tensors holding uint32 values."""
    x = ((a * 0x9E3779B1) & M32) ^ (((b + 0x7F4A7C15) * 0x85EBCA77) & M32) ^ (((c + 0x165667B1) * 0xC2B2AE3D) & M32)
    x = x & M32
    x = x ^ (x >> 16)
    x = (x * 0x7FEB352D) & M32
    x = x ^ (x >> 15)
    x = (x * 0x846CA68B) & M32
    return x ^ (x >> 16)


def keep_threshold(keep):
    return min(int(np.float32(keep) * np.float32(4294967296.0)), M32)


def dropout_scale(seed, p, i, j, L, I, keep, device='cpu'):
    """m / keep [len(i), len(j), I] (float64) of pair p, rows i, columns j: the kernels' counter-based keep decisions."""
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    lo, hi = seed & M32, seed >> 32
    i = torch.as_tensor(np.asarray(i), dtype=torch.int64, device=device)
    j = torch.as_tensor(np.asarray(j), dtype=torch.int64, device=device)
    k = torch.arange(I, dtype=torch.int64, device=device)
    b = (hi ^ ((p * L + i) & M32))[:, None, None]
    c = ((j[:, None] * I + k[None, :]) & M32)[None, :, :]
    h = _hash3(torch.full_like(b, lo), b, c)
    inv = float(np.float32(1.0) / np.float32(keep))
    return torch.where(h < keep_threshold(keep), torch.tensor(inv, dtype=torch.float64, device=device),
                       torch.tensor(0.0, dtype=torch.float64, device=device))


def gelu_tanh(x):
    return 0.5 * x * (1.0 + torch.tanh(C0 * (x + 0.044715 * x ** 3)))


def match_logits(U, V, b1, w2, b2, seq_len, keep=1.0, seed=0, rows=16):
    """U, V [P, L, I], b1 [I], w2 [I], b2 [] float64 tensors -> z [P, L, L] (0 off the candidates), pair by pair and
    `rows` rows at a time.  Differentiable."""
    P, L, I = U.shape
    zs = []
    for p in range(P):
        m = min(max(int(seq_len[p]), 0), L) - 2
        zp = torch.zeros((L, L), dtype=U.dtype, device=U.device)
        for r0 in range(1, m + 1, rows):
            i = np.arange(r0, min(r0 + rows, m + 1))
            j = np.arange(1, m + 1)
            a = gelu_tanh(U[p, i][:, None, :] + V[p, j][None, :, :] + b1)
            if keep < 1.0:
                a = a * dropout_scale(seed, p, i, j, L, I, keep, U.device)
            zz = a @ w2 + b2
            mask = torch.as_tensor(i[:, None] <= j[None, :], device=U.device)
            block = torch.zeros((L, L), dtype=U.dtype, device=U.device)
            block[r0:r0 + len(i), 1:m + 1] = torch.where(mask, zz, torch.zeros_like(zz))
            zp = zp + block
        zs.append(zp)
    return torch.stack(zs) if zs else U.new_zeros((0, L, L))


def bce_loss(z, span_end, seq_len):
    """Mean of BCE-with-logits(z, [j = span_end[p, i]]) over every candidate of the batch, 0 without candidates."""
    P, L, _ = z.shape
    cand = torch.as_tensor(candidates(seq_len, L), device=z.device)
    y = torch.as_tensor(np.asarray(span_end)[:, :, None] == np.arange(L)[None, None, :], dtype=z.dtype, device=z.device)
    el = torch.clamp(z, min=0) - z * y + torch.log1p(torch.exp(-z.abs()))
    n = int(cand.sum())
    return (el * cand).sum() / n if n > 0 else (el * 0).sum()


def sigmoid32(z):
    z = np.float32(z)
    return np.float32(1.0) / (np.float32(1.0) + np.exp(-z, dtype=np.float32))


def project(spans, n, type_tag, o_id, cls_id, sep_id, L):
    """Greedy non-overlapping projection of [(i, j, t, z)] -> tag ids [L]: descending z, then lower type, start, end."""
    tags = np.zeros(L, np.int32)
    if n >= 1:
        tags[1:n - 1] = o_id
        tags[0] = cls_id
        if n >= 2:
            tags[n - 1] = sep_id
    taken = np.zeros(L, bool)
    for i, j, t, _ in sorted(spans, key=lambda s: (-s[3], s[2], s[0], s[1])):
        if taken[i:j + 1].any():
            continue
        taken[i:j + 1] = True
        tags[i] = type_tag[t][0]
        tags[i + 1:j + 1] = type_tag[t][1]
    return tags


def decode(start_logits, end_logits, z, seq_len, type_tag, o_id, cls_id, sep_id, cap):
    """start / end logits [B*T, L, 2] f32 and z [B*T, L, L] f32 -> (pred_ids [B, L], spans [B, cap], probs [B, cap],
    counts [B]); span and prob entries past the count are 0."""
    start_logits, end_logits, z = (np.asarray(a, np.float32) for a in (start_logits, end_logits, z))
    T = len(type_tag)
    P, L, _ = start_logits.shape
    B = P // T
    pred = np.zeros((B, L), np.int32)
    words = np.zeros((B, cap), np.int32)
    probs = np.zeros((B, cap), np.float32)
    counts = np.zeros(B, np.int32)
    for b in range(B):
        n = min(max(int(seq_len[b]), 0), L)
        m = n - 2
        st = start_logits[b * T:(b + 1) * T, :, 1] > start_logits[b * T:(b + 1) * T, :, 0]
        en = end_logits[b * T:(b + 1) * T, :, 1] > end_logits[b * T:(b + 1) * T, :, 0]
        spans = [(i, j, t, float(z[b * T + t, i, j])) for i in range(1, m + 1) for j in range(i, m + 1) for t in range(T)
                 if st[t, i] and en[t, j] and z[b * T + t, i, j] > 0]
        counts[b] = len(spans)
        for o, (i, j, t, zz) in enumerate(spans[:cap]):
            words[b, o] = i | (j + 1) << 12 | t << 24
            probs[b, o] = sigmoid32(zz)
        pred[b] = project(spans, n, type_tag, o_id, cls_id, sep_id, L)
    return pred, words, probs, counts
