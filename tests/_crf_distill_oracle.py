"""Float64 reference of CRF-to-CRF distillation (ner_crf_distill_fwd / _bwd), in torch on any device.

For row b with n_b = clamp(seq_len[b], 0, L), potentials x / tau and transitions T / tau of the teacher (T) and the
student (S), mu the unary and xi the pairwise marginals:

    KL_b = sum_t mu_T[t]·(x_T - x_S)[t] / tau + sum_{t>=1} xi_T[t]·(T_T - T_S) / tau - logZ_T + logZ_S
    d KL_b / d x_S = (mu_S - mu_T) / tau,   d KL_b / d T_S = sum_{t>=1} (xi_S - xi_T) / tau

A term whose teacher marginal is 0 adds 0; n_b = 0 gives KL = 0 and a zero gradient.  `brute_kl` sums over every path
of one row and is what the recursions are checked against.

`distill_ref` returns the student's gradient as a CrfGrad, so `_crf_grad_oracle.grad_errors` judges the kernels with the
existing route bounds: alpha and log Z are those of the larger-magnitude recursion (the size of the float32 rounding),
g_b is the row's coefficient / tau, and trans_scale is S_ij = sum_b |g_b| sum_t (xi_S + xi_T)(i, j).
"""
import itertools
from collections import namedtuple

import numpy as np
import torch

from _crf_grad_oracle import CrfGrad

DistillRef = namedtuple("DistillRef", "kl logz_t logz_s grad kl_scale")


def marginals(x, tr, n):
    """x [B,L,K] f64, tr [K,K] f64, n [B] -> (alpha [B,L,K], logz [B], mu [B,L,K], xi [B,K,K] summed over t >= 1)."""
    B, L, K = x.shape
    dev = x.device
    valid = torch.arange(L, device=dev)[None, :] < n[:, None]
    alpha = torch.empty_like(x)
    alpha[:, 0] = x[:, 0]
    for t in range(1, L):
        alpha[:, t] = x[:, t] + torch.logsumexp(alpha[:, t - 1, :, None] + tr[None], dim=1)
    last = alpha[torch.arange(B, device=dev), (n - 1).clamp(min=0)]
    logz = torch.where(n > 0, torch.logsumexp(last, dim=1), torch.zeros((), dtype=x.dtype, device=dev))
    beta = torch.zeros_like(x)
    for t in range(L - 2, -1, -1):
        rec = torch.logsumexp(tr[None] + (x[:, t + 1] + beta[:, t + 1])[:, None, :], dim=2)
        beta[:, t] = torch.where((t < n - 1)[:, None], rec, torch.zeros_like(rec))
    mu = torch.where(valid[:, :, None], torch.exp(alpha + beta - logz[:, None, None]), torch.zeros_like(x))
    xi = torch.zeros((B, K, K), dtype=x.dtype, device=dev)
    for t in range(1, L):
        pair = torch.exp(alpha[:, t - 1, :, None] + tr[None] + (x[:, t] + beta[:, t])[:, None, :] - logz[:, None, None])
        xi += torch.where(valid[:, t, None, None], pair, torch.zeros_like(pair))
    return alpha, logz, mu, xi


def _times(p, d):
    """p * d with 0 wherever p == 0 (a zero teacher marginal adds nothing, whatever d is)."""
    return torch.where(p > 0, p * d, torch.zeros_like(p))


def distill_ref(t_logits, t_trans, s_logits, s_trans, lens, tau=1.0, g=None):
    dev = s_logits.device
    B, L, K = s_logits.shape
    xt = t_logits.to(device=dev, dtype=torch.float64) / tau
    xs = s_logits.to(torch.float64) / tau
    trt = t_trans.to(device=dev, dtype=torch.float64) / tau
    trs = s_trans.to(device=dev, dtype=torch.float64) / tau
    n = lens.to(device=dev, dtype=torch.long).clamp(0, L)
    g = torch.ones(B, dtype=torch.float64, device=dev) if g is None else g.to(device=dev, dtype=torch.float64)
    at, lzt, mut, xit = marginals(xt, trt, n)
    as_, lzs, mus, xis = marginals(xs, trs, n)
    kl = (_times(mut, xt - xs).sum((1, 2)) + _times(xit, (trt - trs)[None]).sum((1, 2))) - lzt + lzs
    kl = torch.where(n > 0, kl, torch.zeros_like(kl))
    # M_b = sum_t mu_T |x_T - x_S| + sum xi_T |T_T - T_S|: the size of the terms KL_b sums, against which the float32
    # rounding of log-domain marginals is judged
    kl_scale = _times(mut, (xt - xs).abs()).sum((1, 2)) + _times(xit, (trt - trs).abs()[None]).sum((1, 2))
    gt = g / tau
    d_logits = gt[:, None, None] * (mus - mut)
    d_trans = torch.einsum("b,bij->ij", gt, xis - xit)
    scale = torch.einsum("b,bij->ij", gt.abs(), xis + xit)
    fa = torch.where(torch.isfinite(at), at, torch.zeros_like(at))
    alpha = torch.where(fa.abs() > as_.abs(), fa, as_)
    logz = torch.where(lzt.abs() > lzs.abs(), lzt, lzs)
    return DistillRef(kl, lzt, lzs, CrfGrad(alpha, logz, d_logits, d_trans, gt, n, scale), kl_scale)


def brute_kl(xt, trt, xs, trs, tau=1.0):
    """KL(p_T || p_S) of one row (x [n,K], tr [K,K], numpy float64) by summing over all K^n paths."""
    n, K = xs.shape
    paths = np.array(list(itertools.product(range(K), repeat=n)))
    rows = np.arange(n)

    def scores(x, tr):
        s = x[rows[None, :], paths].sum(1)
        if n > 1:
            s = s + tr[paths[:, :-1], paths[:, 1:]].sum(1)
        return s / tau

    st, ss = scores(xt, trt), scores(xs, trs)
    lzt = np.logaddexp.reduce(st)
    lzs = np.logaddexp.reduce(ss)
    pt = np.exp(st - lzt)
    live = pt > 0
    return float((pt[live] * ((st[live] - lzt) - (ss[live] - lzs))).sum())
