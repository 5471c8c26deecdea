"""Float64 forward-backward of the partial-annotation CRF (ner_crf_partial_loglik_fwd / _bwd), in torch on any device.

For row b with n_b = clamp(seq_len[b], 0, L) and allowed sets A_t = {j < K : bit j of label_mask[b, t]}:

    ll_b = logZ_A - logZ,   d ll_b / d x[t][j] = P_A(y_t = j) - P(y_t = j),
    d ll_b / d trans[i][j] = sum_t P_A(y_{t-1} = i, y_t = j) - P(y_{t-1} = i, y_t = j)

logZ_A is the partition function of the logits with every disallowed tag at -inf, so both halves are `crf_grad_ref`
(tests/_crf_grad_oracle.py) run twice: the gold-path terms of the two runs cancel.  n_b = 0 gives ll = 0; an empty A_t at
some t < n_b, or sets that only -inf transitions join, give ll = -inf and a zero gradient (the row is dropped from
d_trans).

`partial_grad_ref` returns a CrfGrad, so `assert_grads_close` judges the kernels with the existing bounds: alpha and
log Z are those of the larger-magnitude recursion (the size of the float32 rounding) and trans_scale is
S_ij = sum_b |g_b| sum_t (P_A + P)(pair i, j).
"""
import itertools
from collections import namedtuple

import numpy as np
import torch

from _crf_grad_oracle import EPS32, CrfGrad, crf_grad_ref

PartialRef = namedtuple("PartialRef", "ll logz_a logz empty grad trans_unit")


def allowed_tags(label_mask, K):
    """[B, L] int32 bitmasks -> [B, L, K] bool (bit 31 is the sign bit of an int32; bits >= K are ignored)."""
    m = label_mask.to(torch.int64) & 0xFFFFFFFF
    return ((m[..., None] >> torch.arange(K, device=m.device)) & 1).bool()


def partial_grad_ref(x, label_mask, lens, trans, g=None):
    dev = x.device
    B, L, K = x.shape
    x = x.to(torch.float64)
    allowed = allowed_tags(label_mask.to(dev), K)
    n = lens.to(device=dev, dtype=torch.long).clamp(0, L)
    valid = torch.arange(L, device=dev)[None, :] < n[:, None]
    empty = (valid & ~allowed.any(-1)).any(1)
    g = torch.ones(B, dtype=torch.float64, device=dev) if g is None else g.to(device=dev, dtype=torch.float64)
    zeros = torch.zeros((B, L), dtype=torch.int32, device=dev)
    # rows with no path inside the sets (an empty set, or sets only -inf transitions join) have Z_A = 0
    xa = torch.where(allowed | empty[:, None, None], x, torch.full_like(x, -float("inf")))
    empty = empty | ((crf_grad_ref(xa, zeros, lens, trans).logz == -float("inf")) & (n > 0))
    g = torch.where(empty, torch.zeros_like(g), g)
    xa = torch.where(allowed | empty[:, None, None], x, torch.full_like(x, -float("inf")))
    ra = crf_grad_ref(xa, zeros, lens, trans, g)
    rf = crf_grad_ref(x, zeros, lens, trans, g)

    ll = torch.where(empty, torch.full_like(ra.logz, -float("inf")), ra.logz - rf.logz)
    d_logits = rf.d_logits - ra.d_logits
    d_trans = rf.d_trans - ra.d_trans
    # both runs counted the all-zeros gold path into S[0][0]: take it out again
    scale = ra.trans_scale + rf.trans_scale
    scale[0, 0] -= 2 * (g.abs() * (n - 1).clamp(min=0)).sum()
    fa = torch.where(torch.isfinite(ra.alpha), ra.alpha, torch.zeros_like(ra.alpha))
    alpha = torch.where(fa.abs() > rf.alpha.abs(), fa, rf.alpha)
    logz = torch.where(ra.logz.abs() > rf.logz.abs(), ra.logz, rf.logz)
    grad = CrfGrad(alpha, logz, d_logits, d_trans, g, n, scale.clamp(min=0))
    # U_ij = sum_b |g_b| EPS32 (1 + |log Z_b| + max |alpha_b|) S_b,ij: the float32 rounding of log-domain marginals.  A
    # kernel holds log Z and alpha as float32 logarithms, so every marginal of row b carries a relative error of that
    # size, and it does not average out over the row's steps (the error of log Z is common to all of them)
    valid3 = valid[:, :, None] & torch.isfinite(alpha)
    amax = torch.where(valid3, alpha.abs(), torch.zeros_like(alpha)).reshape(B, -1).max(dim=1).values
    r = EPS32 * (1 + logz.abs().nan_to_num(0, 0, 0) + amax)
    ua = crf_grad_ref(xa, zeros, lens, trans, g.abs() * r).trans_scale
    uf = crf_grad_ref(x, zeros, lens, trans, g.abs() * r).trans_scale
    unit = ua + uf
    unit[0, 0] -= 2 * (g.abs() * r * (n - 1).clamp(min=0)).sum()
    return PartialRef(ll, ra.logz, rf.logz, empty, grad, unit.clamp(min=0))


def step_pair(x, label_mask, trans, g, t):
    """sum_b g_b (P_A - P)(y_{t-1} = i, y_t = j) of full-length rows: the share of step t in d_trans (what a kernel that
    skipped that step would miss).  beta comes from the forward recursion of the reversed rows."""
    B, L, K = x.shape
    x = x.to(torch.float64)
    tr = trans.to(device=x.device, dtype=torch.float64)
    xa = torch.where(allowed_tags(label_mask.to(x.device), K), x, torch.full_like(x, -float("inf")))
    lens = torch.full((B,), L, dtype=torch.int32, device=x.device)
    zeros = torch.zeros((B, L), dtype=torch.int32, device=x.device)
    out = 0
    for xx, sign in ((xa, 1.0), (x, -1.0)):
        fwd = crf_grad_ref(xx, zeros, lens, tr)
        rev = crf_grad_ref(xx.flip(1), zeros, lens, tr.t())          # alpha_rev[L-1-t] = x_t + beta_t
        p = torch.exp(fwd.alpha[:, t - 1, :, None] + tr[None] + rev.alpha[:, L - 1 - t, None, :]
                      - fwd.logz[:, None, None])
        out = out + sign * torch.einsum("b,bij->ij", g.to(torch.float64), p)
    return out


def brute_force_partial(x, allowed, trans, n):
    """ONE sequence by enumerating all K^n paths: (ll, P_A - P [n, K], sum_t (P_A - P) pairs [K, K])."""
    x = np.asarray(x, dtype=np.float64)
    tr = np.asarray(trans, dtype=np.float64)
    K = x.shape[1]
    if n == 0:
        return 0.0, np.zeros((0, K)), np.zeros((K, K))
    paths = list(itertools.product(range(K), repeat=n))
    score = np.array([sum(x[t, p[t]] for t in range(n)) + sum(tr[p[t - 1], p[t]] for t in range(1, n)) for p in paths])
    inside = np.array([all(allowed[t][p[t]] for t in range(n)) for p in paths])
    if not inside.any():
        return -np.inf, np.zeros((n, K)), np.zeros((K, K))

    def posterior(sel):
        s = np.where(sel, score, -np.inf)
        m = s.max()
        w = np.exp(s - m)
        return m + np.log(w.sum()), w / w.sum()

    lza, wa = posterior(inside)
    lzf, wf = posterior(np.ones_like(inside))
    unary, pair = np.zeros((n, K)), np.zeros((K, K))
    for p, d in zip(paths, wa - wf):
        for t in range(n):
            unary[t, p[t]] += d
            if t:
                pair[p[t - 1], p[t]] += d
    return lza - lzf, unary, pair


def _log_norm(x, n, tr):
    alpha = x[:, 0]
    for t in range(1, x.shape[1]):
        nxt = x[:, t] + torch.logsumexp(alpha[:, :, None] + tr[None], dim=1)
        alpha = torch.where((t < n)[:, None], nxt, alpha)
    return torch.where(n > 0, torch.logsumexp(alpha, dim=1), torch.zeros_like(alpha[:, 0]))


def partial_ll_torch(logits, label_mask, lens, trans):
    """Differentiable (autograd) ll_b of rows whose allowed sets are all non-empty: the loss of a plugin graph."""
    K = logits.shape[-1]
    allowed = allowed_tags(label_mask.to(logits.device), K)
    n = lens.to(device=logits.device, dtype=torch.long).clamp(0, logits.shape[1])
    xa = torch.where(allowed, logits, torch.full_like(logits, -float("inf")))
    return _log_norm(xa, n, trans) - _log_norm(logits, n, trans)
