"""numpy restatement of the bert_mrc glue (include/ner_b200.h: ner_mrc_pairs, ner_mrc_merge): the query/context pairs,
their per-type BIO labels, the sentence alignment and the cross-type tag merge."""
import numpy as np


def mrc_pairs(token_ids, seq_len, query_ids, query_len, type_tag, L2, sep_id, label_ids=None):
    """-> dict(ids, segment_ids, mask [B*T, L2], seq_len [B*T], align [B*T*L], labels [B*T, L] | None), int32."""
    token_ids = np.asarray(token_ids)
    B, L = token_ids.shape
    T, Qmax = np.asarray(query_ids).reshape(len(query_len), -1).shape
    query_ids = np.asarray(query_ids).reshape(T, Qmax)
    ids = np.zeros((B * T, L2), np.int32)
    seg = np.zeros((B * T, L2), np.int32)
    mask = np.zeros((B * T, L2), np.int32)
    plen = np.zeros(B * T, np.int32)
    align = np.zeros((B * T, L), np.int32)
    labels = None if label_ids is None else np.zeros((B * T, L), np.int32)
    for b in range(B):
        n_sent = min(max(int(seq_len[b]), 0), L)
        for t in range(T):
            p = b * T + t
            q = min(max(int(query_len[t]), 0), Qmax)
            plen[p] = n_sent
            if n_sent > 0:
                row = [token_ids[b, 0]] + list(query_ids[t, :q]) + [sep_id] + list(token_ids[b, 1:n_sent])
                n = len(row)
                assert n == q + 1 + n_sent
                ids[p, :n] = row
                mask[p, :n] = 1
                seg[p, q + 2:n] = 1
            for s in range(L):
                align[p, s] = p * L2 + (0 if s == 0 else q + 1 + s)
                if labels is not None and s < n_sent:
                    tag = int(label_ids[b, s])
                    labels[p, s] = 1 if tag == type_tag[t][0] else 2 if tag == type_tag[t][1] else 0
    return dict(ids=ids, segment_ids=seg, mask=mask, seq_len=plen, align=align.reshape(-1), labels=labels)


def type_scores(z):
    """z [..., 3] float32 -> (first argmax [...], z[a] - logsumexp(z) in float32 [...])."""
    z = np.asarray(z, np.float32)
    a = np.argmax(z, -1)
    m = np.take_along_axis(z, a[..., None], -1)
    e = np.exp(z - m).astype(np.float32)
    s = (e[..., 0] + e[..., 1]) + e[..., 2]
    return a, -np.log(s).astype(np.float32)


def mrc_merge(logits, seq_len, type_tag, o_id, cls_id, sep_id):
    """logits [B*T, L, 3] -> pred_ids [B, L] int32 (the rule of ner_mrc_merge), and the decision margin [B, L]: the
    smaller of the closest top-1 / top-2 logit gap of any type and the winner's score lead over the runner-up claim
    (inf where the tag is fixed or nothing competes)."""
    logits = np.asarray(logits, np.float32)
    T = len(type_tag)
    BT, L, _ = logits.shape
    B = BT // T
    z = logits.reshape(B, T, L, 3)
    a, score = type_scores(z)
    top2 = np.sort(z, -1)
    gap = (top2[..., 2].astype(np.float64) - top2[..., 1]).min(1)           # [B, L]
    pred = np.zeros((B, L), np.int32)
    margin = np.full((B, L), np.inf)
    for b in range(B):
        n = min(max(int(seq_len[b]), 0), L)
        for s in range(n):
            if s == 0:
                pred[b, s] = cls_id
            elif s == n - 1:
                pred[b, s] = sep_id
            else:
                margin[b, s] = gap[b, s]
                cand = [t for t in range(T) if a[b, t, s] != 0]
                if not cand:
                    pred[b, s] = o_id
                    continue
                best = max(cand, key=lambda t: (score[b, t, s], -t))
                pred[b, s] = type_tag[best][a[b, best, s] - 1]
                others = [score[b, t, s] for t in cand if t != best]
                if others:
                    margin[b, s] = min(margin[b, s], float(score[b, best, s]) - max(float(o) for o in others))
    return pred, margin
