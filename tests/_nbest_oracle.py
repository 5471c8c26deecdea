"""Numpy fp32 list Viterbi: the N best CRF paths under the rule of ner_crf_viterbi_nbest, followed literally.

Row b decodes n = min(max(seq_len[b], 1), L) positions.  Each (t, j) keeps up to N entries (score, i, r): the candidates
(predecessor tag i, its rank r) are ordered by s_{t-1}[i][r] + trans[i][j] descending (the sum ner_crf_viterbi compares),
then lower i, then lower r, and the entry's score is that sum + x[t][j].  The lists at n - 1 are merged by score
descending, lower last tag, lower rank; the first N are backtracked.  All arithmetic is float32 in the order above.
"""
import itertools

import numpy as np

f32 = np.float32


def path_score(x, trans, path):
    """Sequential fp32 score of one path: s_0 = x[0, y_0], s_t = (s_{t-1} + trans[y_{t-1}, y_t]) + x[t, y_t]."""
    s = f32(x[0, path[0]])
    for t in range(1, len(path)):
        s = f32(f32(s + trans[path[t - 1], path[t]]) + x[t, path[t]])
    return s


def nbest(x, trans, seq_len, N):
    """x [B, L, K], trans [K, K], seq_len [B] -> (tags [B, N, L] int32, scores [B, N] float32, counts [B] int32), with
    zero tags past n and in empty ranks, and score -inf in empty ranks."""
    x = np.asarray(x, dtype=f32)
    trans = np.asarray(trans, dtype=f32)
    B, L, K = x.shape
    n = np.clip(np.asarray(seq_len, dtype=np.int64), 1, L)
    lists = x[:, 0, :, None].copy()            # [B, K, cnt]: scores of each tag's list at the current step
    cnt = 1
    back = [None]                              # back[t]: (i, r) [B, K, cnt_t] of the entries at step t
    final = [None] * B
    for b in np.nonzero(n == 1)[0]:
        final[b] = lists[b]
    for t in range(1, int(n.max())):
        cnew = min(N, cnt * K)
        pre = (lists[:, :, :, None] + trans[None, :, None, :]).astype(f32).reshape(B, K * cnt, K)   # index i*cnt + r
        order = np.argsort(-pre, axis=1, kind='stable')[:, :cnew, :]                                # ties: lower (i, r)
        best = np.take_along_axis(pre, order, axis=1)                                               # [B, cnew, K]
        lists = (best + x[:, t, None, :]).astype(f32).transpose(0, 2, 1).copy()                     # [B, K, cnew]
        back.append(((order // cnt).transpose(0, 2, 1), (order % cnt).transpose(0, 2, 1)))
        cnt = cnew
        for b in np.nonzero(n == t + 1)[0]:
            final[b] = lists[b]
    tags = np.zeros((B, N, L), dtype=np.int32)
    scores = np.full((B, N), -np.inf, dtype=f32)
    counts = np.zeros((B,), dtype=np.int32)
    for b in range(B):
        fl = final[b]                                   # [K, c]
        c = fl.shape[1]
        flat = fl.reshape(-1)                           # index j*c + r
        order = np.argsort(-flat, kind='stable')[:N]
        counts[b] = len(order)
        for k, o in enumerate(order):
            y, r = int(o) // c, int(o) % c
            scores[b, k] = flat[o]
            for t in range(int(n[b]) - 1, 0, -1):
                tags[b, k, t] = y
                bi, br = back[t]
                y, r = int(bi[b, y, r]), int(br[b, y, r])
            tags[b, k, 0] = y
    return tags, scores, counts


def all_paths(x, trans, n):
    """Every one of the K^n paths of one sequence's first n positions with its sequential fp32 score, best first
    (a stable sort of the lexicographic enumeration)."""
    x = np.asarray(x, dtype=f32)
    trans = np.asarray(trans, dtype=f32)
    K = x.shape[1]
    paths = np.array(list(itertools.product(range(K), repeat=n)), dtype=np.int64).reshape(-1, n)
    s = x[0, paths[:, 0]].astype(f32)
    for t in range(1, n):
        s = ((s + trans[paths[:, t - 1], paths[:, t]]).astype(f32) + x[t, paths[:, t]]).astype(f32)
    order = np.argsort(-s, kind='stable')
    return paths[order], s[order]
