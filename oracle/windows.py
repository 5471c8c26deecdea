"""Plain restatement of the BERT plugins' document mode (chinesener_b200/windows.py, csrc/window.cu): window starts,
window tokens and the owner of every document position, written as loops over the definition (run_squad.py's doc_stride
windows and _check_is_max_context), plus a windowed encoder: nn.bert_encoder per window, stitched by owner."""
import numpy as np
import torch

from . import nn

_bert_encoder = nn.bert_encoder      # the per-window encoder, bound here so a test may patch nn.bert_encoder with windowed()


def window_starts(n, W, S):
    """Content offsets a_k of the windows of a document with n tokens ([0] for n <= W, [] for n = 0)."""
    if n <= 0:
        return []
    if n <= W:
        return [0]
    C, m = W - 2, n - 2
    starts, a = [], 0
    while True:
        starts.append(min(a, m - C))
        if a + C >= m:
            return starts
        a += S


def window_positions(n, W, S):
    """[nw, len] doc positions of each window's tokens: the document itself for n <= W, else [0, 1 + a .. a + C, n - 1]."""
    if n <= W:
        return np.arange(n, dtype=np.int64).reshape(1 if n > 0 else 0, n)
    C = W - 2
    a = np.array(window_starts(n, W, S), dtype=np.int64)[:, None]
    return np.concatenate([np.zeros_like(a), 1 + a + np.arange(C), np.full_like(a, n - 1)], axis=1)


def owners(n, W, S):
    """-> [(window k, row p)] for doc positions 0 .. n - 1: [CLS] row 0 of window 0, [SEP] row W - 1 of the last window,
    content index c the window with the largest min(c - a_k, a_k + C - 1 - c) (max context), the lowest k on a tie."""
    if n <= W:
        return [(0, t) for t in range(n)]
    C = W - 2
    a = np.array(window_starts(n, W, S))
    c = np.arange(n - 2)
    # the windows holding c are consecutive from the first one that ends after c, and there are at most C // S + 1
    first = np.searchsorted(a + C, c, side='right')
    k = first[:, None] + np.arange(min(len(a), C // S + 1))[None, :]
    ak = a[np.minimum(k, len(a) - 1)]
    holds = (k < len(a)) & (ak <= c[:, None]) & (c[:, None] < ak + C)
    score = np.where(holds, np.minimum(c[:, None] - ak, ak + C - 1 - c[:, None]), -1)
    j = score.argmax(1)                                   # first maximum: the lowest window on a tie
    kk = k[np.arange(len(c)), j]
    return [(0, 0)] + [(int(x), int(y - a[x] + 1)) for x, y in zip(kk, c)] + [(len(a) - 1, W - 1)]


def plan(lengths, W, S):
    """Batch plan -> dict(pos [NW, W] doc position per window row (-1 at [PAD]), doc [NW] document of each window,
    src_padded / src_packed [sum n] the owner row of each doc token in the window-padded / window-packed layouts)."""
    pos, doc, src_padded, src_packed = [], [], [], []
    tok = 0
    for b, n in enumerate(lengths):
        n = int(n)
        w0 = len(pos)
        wins = window_positions(n, W, S)
        for p in wins.tolist():
            pos.append(p + [-1] * (W - len(p)))
            doc.append(b)
        for k, p in owners(n, W, S):
            src_padded.append((w0 + k) * W + p)
            src_packed.append(tok + (p if n <= W else k * W + p))
        tok += n if n <= W else len(wins) * W
    return dict(pos=np.array(pos, dtype=np.int64).reshape(-1, W), doc=np.array(doc, dtype=np.int64),
                src_padded=np.array(src_padded, dtype=np.int64), src_packed=np.array(src_packed, dtype=np.int64))


def windowed(W, S):
    """-> an nn.bert_encoder replacement: a batch with L > W runs nn.bert_encoder on each document's windows and takes
    every token's row from its owner window (zero rows at [PAD]); differentiable, so autograd reaches the weights through
    the windows.  L <= W is nn.bert_encoder itself."""
    def encoder(w, input_ids, input_mask, segment_ids, **kw):
        B, L = input_ids.shape
        if L <= W:
            return _bert_encoder(w, input_ids, input_mask, segment_ids, **kw)
        lengths = [int(v) for v in input_mask.sum(1)]
        pl = plan(lengths, W, S)
        pos, doc = torch.from_numpy(pl['pos']), torch.from_numpy(pl['doc'])
        real = pos >= 0
        gather = lambda x: torch.where(real, x[doc[:, None], pos.clamp(min=0)], torch.zeros_like(pos)).to(x.dtype)
        seg = None if segment_ids is None else gather(segment_ids.long())
        seq = _bert_encoder(w, gather(input_ids.long()), real.to(torch.int32), seg, **kw)       # [NW, W, H]
        flat = seq.reshape(-1, seq.shape[-1])
        rows = flat[torch.from_numpy(pl['src_padded'])]
        doc_rows = torch.cat([torch.arange(n) + b * L for b, n in enumerate(lengths)])
        return flat.new_zeros(B * L, flat.shape[-1]).index_copy(0, doc_rows, rows).view(B, L, -1)
    return encoder
