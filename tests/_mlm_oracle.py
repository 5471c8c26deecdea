"""numpy / float64 restatements of the masked-LM kernels (ner_mlm_mask, ner_vocab_xent) and head (chinesener_b200/mlm.py),
the checkers of the GPU tests."""
import numpy as np
import torch

M32 = 0xFFFFFFFF


def hash3(a, b, c):
    """common.cuh hash3 on uint32 (numpy arrays or ints)."""
    with np.errstate(over="ignore"):
        return _hash3(*(np.asarray(x, dtype=np.uint64) & np.uint64(M32) for x in (a, b, c)))


def _hash3(a, b, c):
    x = ((a * 0x9E3779B1) & M32) ^ (((b + 0x7F4A7C15) & M32) * 0x85EBCA77 & M32) ^ (((c + 0x165667B1) & M32) * 0xC2B2AE3D & M32)
    x ^= x >> 16
    x = (x * 0x7FEB352D) & M32
    x ^= x >> 15
    x = (x * 0x846CA68B) & M32
    x ^= x >> 16
    return x


def mask_hash(seed, k, b, t):
    return hash3((seed + k * 0x9E3779B9) & M32, ((seed >> 32) & M32) ^ b, t)


def google_budget(n, p, max_pred):
    """create_pretraining_data.py's num_to_predict over n = len(tokens) (no candidates for n <= 2)."""
    if n <= 2:
        return 0
    return min(max_pred, max(1, int(round(n * p))))


def words_of_row(n, word_start_row):
    """-> list of (first position, length) of the words of a row with n tokens."""
    words = []
    for t in range(1, n - 1):
        if t == 1 or word_start_row is None or word_start_row[t]:
            words.append([t, 1])
        else:
            words[-1][1] += 1
    return [tuple(w) for w in words]


def mask_row(tokens, n, word_start_row, k, seed, b, V, mask_id):
    """-> (masked row, chosen positions ascending) of one row, as ner_mlm_mask."""
    L = len(tokens)
    n = min(max(int(n), 0), L)
    words = words_of_row(n, word_start_row)
    order = sorted(words, key=lambda w: (int(mask_hash(seed, 0, b, w[0])), w[0]))
    taken, chosen = 0, []
    for s, ln in order:
        if taken >= k:
            break
        if taken + ln <= k:
            taken += ln
            chosen.extend(range(s, s + ln))
    chosen.sort()
    out = np.array(tokens, dtype=np.int64)
    for t in chosen:
        u = int(mask_hash(seed, 1, b, t)) >> 8
        if u * 5 < 4 << 24:
            out[t] = mask_id
        elif u * 10 < 9 << 24:
            out[t] = (int(mask_hash(seed, 2, b, t)) * V) >> 32
    return out, chosen


def mlm_mask(token_ids, seq_len, word_start, offsets, seed, V, mask_id):
    """-> (masked_ids [B,L], positions [M], labels [M]) of ner_mlm_mask."""
    B, L = token_ids.shape
    masked = np.array(token_ids, dtype=np.int64)
    M = int(offsets[-1])
    pos, lab = np.zeros(M, np.int64), np.zeros(M, np.int64)
    for b in range(B):
        k = max(int(offsets[b + 1]) - int(offsets[b]), 0)
        row, chosen = mask_row(token_ids[b], seq_len[b], None if word_start is None else word_start[b], k, seed, b, V,
                               mask_id)
        masked[b] = row
        o = int(offsets[b])
        for i in range(k):
            if i < len(chosen):
                pos[o + i], lab[o + i] = b * L + chosen[i], token_ids[b, chosen[i]]
            else:
                pos[o + i], lab[o + i] = b * L, -1
    return masked, pos, lab


def vocab_xent(logits, labels, V, d_loss=1.0):
    """float64 ner_vocab_xent -> (loss, count, correct, pred [M], d_logits [M, ld])."""
    z = np.asarray(logits, np.float64)
    M, ld = z.shape
    zv = z[:, :V]
    pred = zv.argmax(1) if M else np.zeros(0, np.int64)
    y = np.asarray(labels)
    cnt = (y >= 0) & (y < V)
    count = int(cnt.sum())
    d = np.zeros_like(z)
    loss = 0.0
    if count:
        m = zv.max(1, keepdims=True)
        e = np.exp(zv - m)
        s = e.sum(1, keepdims=True)
        lse = (m + np.log(s))[:, 0]
        rows = np.nonzero(cnt)[0]
        loss = float((lse[rows] - zv[rows, y[rows]]).sum() / count)
        g = e / s
        g[rows, y[rows]] -= 1.0
        d[rows, :V] = g[rows] * (d_loss / count)
    correct = int((cnt & (pred == y)).sum())
    return loss, count, correct, pred, d


def head_logits(h, w, V, dtype=torch.float64, gelu_variant="tanh"):
    """get_masked_lm_output on gathered rows h [M, H] -> logits [M, V]."""
    from oracle import nn as onn
    g = lambda n: w[n].to(dtype)
    t = onn.gelu(h @ g("cls/predictions/transform/dense/kernel") + g("cls/predictions/transform/dense/bias"), gelu_variant)
    t = onn.layer_norm(t, g("cls/predictions/transform/LayerNorm/gamma"), g("cls/predictions/transform/LayerNorm/beta"), 1e-12)
    return t @ g("bert/embeddings/word_embeddings")[:V].T + g("cls/predictions/output_bias")


def masked_lm_loss(logits, labels):
    """Exact mean CE over the labels in [0, V) (torch, differentiable)."""
    keep = labels >= 0
    lp = torch.log_softmax(logits, -1)
    return -(lp[keep, labels[keep]]).sum() / max(int(keep.sum()), 1)
