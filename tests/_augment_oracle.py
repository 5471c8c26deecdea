"""Pure-Python / numpy restatement of ner_augment_rows and ner_vocab_sample (include/ner_b200.h), the checker of the GPU
tests.  Hashes are _mlm_oracle.hash3; rows are walked in plain Python so the rules read as stated."""
import numpy as np

from _mlm_oracle import M32, hash3

BUDGET = 20
ROW, MR_PICK, MR_DRAW, LW_PICK, LW_DRAW, SIS_PICK, SIS_KEY, MLM_PICK, GUMBEL = range(9)


def h(seed, k, b, t):
    return int(hash3((seed + k * 0x9E3779B9) & M32, ((seed >> 32) & M32) ^ b, t))


def thr(p):
    return int(np.float32(p) * np.float32(16777216.0))


def drawn(hv, p):
    return (hv >> 8) < thr(p)


def pick(hv, n):
    return (hv * n) >> 32


def segments(tags, cls, type_tag):
    """-> list of (start, length) of a row's segments: a mention (B-x then its I-x run), a maximal run of O, or any other
    single token (a stray I-x, a special tag)."""
    K = len(cls)
    c = [int(cls[y]) if 0 <= y < K else 0 for y in tags]
    segs, t, n = [], 0, len(tags)
    while t < n:
        e = t
        if c[t] == 1:
            while e + 1 < n and c[e + 1] == 1:
                e += 1
        elif c[t] >= 2 and c[t] % 2 == 0:
            inside = int(type_tag[(c[t] - 2) // 2][1])
            while e + 1 < n and inside >= 0 and tags[e + 1] == inside:
                e += 1
        segs.append((t, e - t + 1))
        t = e + 1
    return segs


def augment_row(b, toks, tags, n, L, pool, probs, seed, mask_id=-1, mlm=False):
    """One augmented row -> (tokens, tags, mlm_ids or None, positions list).  probs = (row, mr, lwtr, sis, mlm)."""
    cls, tt = pool.tag_class, pool.type_tag
    K = len(cls)
    cl = lambda y: int(cls[y]) if 0 <= y < K else 0
    toks, tags = [int(x) for x in toks[:n]], [int(y) for y in tags[:n]]
    _, p_mr, p_lw, p_sis, p_mlm = probs
    if p_mr > 0:
        out_t, out_y, cur, s = [], [], n, 0
        while s < n:
            y = tags[s]
            c = cl(y)
            if c < 2 or c % 2:
                out_t.append(toks[s])
                out_y.append(y)
                s += 1
                continue
            x = (c - 2) // 2
            inside = int(tt[x][1])
            e = s
            while e + 1 < n and tags[e + 1] == inside:
                e += 1
            ln = e - s + 1
            done = False
            if drawn(h(seed, MR_PICK, b, s), p_mr):
                lo, hi = int(pool.mention_type_off[x]), int(pool.mention_type_off[x + 1])
                if hi > lo:
                    j = lo + pick(h(seed, MR_DRAW, b, s), hi - lo)
                    m = pool.mention_tokens[pool.mention_tok_off[j]:pool.mention_tok_off[j + 1]]
                    nl = len(m)
                    if nl >= 1 and (nl == 1 or inside >= 0) and cur - ln + nl <= L:
                        out_t += [int(v) for v in m]
                        out_y += [y] + [inside] * (nl - 1)
                        cur += nl - ln
                        done = True
            if not done:
                out_t += toks[s:e + 1]
                out_y += tags[s:e + 1]
            s = e + 1
        toks, tags = out_t, out_y
    n = len(toks)
    if p_lw > 0:
        for t in range(n):
            y = tags[t]
            if cl(y) >= 1 and drawn(h(seed, LW_PICK, b, t), p_lw):
                lo, hi = int(pool.tag_tok_off[y]), int(pool.tag_tok_off[y + 1])
                if hi > lo:
                    toks[t] = int(pool.tag_tokens[lo + pick(h(seed, LW_DRAW, b, t), hi - lo)])
    if p_sis > 0:
        new = list(toks)
        for s, ln in segments(tags, cls, tt):
            if ln >= 2 and drawn(h(seed, SIS_PICK, b, s), p_sis):
                order = sorted(range(s, s + ln), key=lambda t: (h(seed, SIS_KEY, b, t), t))
                for i, src in enumerate(order):
                    new[s + i] = toks[src]
        toks = new
    mids, pos = None, []
    if mlm:
        mids = list(toks)
        for t in range(n):
            if len(pos) < BUDGET and p_mlm > 0 and cl(tags[t]) == 1 and drawn(h(seed, MLM_PICK, b, t), p_mlm):
                pos.append(t)
                mids[t] = mask_id
    return toks, tags, mids, pos


def augment_rows(token_ids, label_ids, seq_len, mask, segment_ids, pool, probs, seed, mask_id=-1, mlm=False):
    """Batch form -> dict like ops.augment_rows (numpy int32)."""
    B, L = token_ids.shape
    out = {k: np.array(v, np.int32) for k, v in (('token_ids', token_ids), ('label_ids', label_ids), ('mask', mask),
                                                 ('segment_ids', segment_ids), ('seq_len', seq_len))}
    if mlm:
        out['mlm_ids'] = np.array(token_ids, np.int32)
        out['mlm_positions'] = np.full((B, BUDGET), -1, np.int32)
    for b in range(B):
        if not drawn(h(seed, ROW, b, 0), probs[0]):
            continue
        n0 = min(max(int(seq_len[b]), 0), L)
        toks, tags, mids, pos = augment_row(b, token_ids[b], label_ids[b], n0, L, pool, probs, seed, mask_id, mlm)
        n = len(toks)
        out['token_ids'][b] = toks + [pool.pad_id] * (L - n)
        out['label_ids'][b] = tags + [pool.pad_tag] * (L - n)
        out['mask'][b] = [1] * n + [0] * (L - n)
        out['segment_ids'][b] = 0
        out['seq_len'][b] = n
        if mlm:
            out['mlm_ids'][b] = mids + [pool.pad_id] * (L - n)
            out['mlm_positions'][b, :len(pos)] = [b * L + t for t in pos]
    return out


def gumbel_scores(logits_row, V, eligible, orig, pos, temperature, seed):
    """float64 scores of ner_vocab_sample's Gumbel-max draw at one slot (-inf where excluded)."""
    j = np.arange(V)
    hv = hash3((seed + GUMBEL * 0x9E3779B9) & M32, ((seed >> 32) & M32) ^ pos, j)
    u = ((hv >> np.uint64(9)).astype(np.float64) + 0.5) / 2.0 ** 23
    s = np.asarray(logits_row[:V], np.float64) / temperature - np.log(-np.log(u))
    ok = (np.asarray(eligible[:V]) != 0) & (j != orig)
    return np.where(ok, s, -np.inf)
