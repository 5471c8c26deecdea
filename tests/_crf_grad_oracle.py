"""Batched float64 forward-backward of the CRF log-likelihood, in torch on any device, and the comparator the CRF
gradient tests judge the CUDA kernels with.

`crf_grad_ref` returns alpha, log Z and the gradient of sum_b g_b * ll_b with respect to the logits and the transition
matrix, under the kernels' conventions: lengths clamped to [0, L], a length <= 0 gives log Z = 0 and a zero gradient,
tags clamped to [0, K-1], -inf transitions allowed.  d_trans is accumulated one step at a time, so memory stays at
O(B*K^2) and a GPU can take batches of tens of thousands of rows in float64.
"""
from collections import namedtuple

import torch

CrfGrad = namedtuple("CrfGrad", "alpha logz d_logits d_trans g lens trans_scale")

EPS32 = 2.0 ** -23

# (rtol, c_dl, tol_s) of each backward kernel (routes as bwd_route in test_crf_bwd_gpu.py names them), checked by
# assert_grads_close:
#     |d_logits - ref| <= rtol |ref| + c_dl u_b,   u_b = |g_b| EPS32 (1 + |log Z_b| + max |alpha_b|) sqrt(len_b)
#     |d_trans - ref|  <= tol_s S_ij
# The kernels hold alpha, beta and log Z as float32 logarithms: a marginal exp(alpha + beta - log Z) carries the
# rounding of values that large, accumulated over len_b steps, so its error grows with both (a 512-step row errs
# ~100x more than a 24-step one, relative to |g_b|).  The numbers are set from H100 runs of test_crf_bwd_gpu.py.
TOL = {
    "lanes": (0.0, 1.0, 1e-4),
    "nt32": (0.0, 2.0, 2e-5),
    "nt64": (0.0, 2.0, 2e-6),
}

SMALL_B = 4096          # NER_CRF_SMALL_B, crf_common.cuh


def bwd_smem_bytes(K, NT, nf):
    """bwd_smem_bytes<K, NT, NF> of crf_common.cuh: transitions x3, row maxima, row lengths, and a 2-stage ring of nf
    8-step float chunks (logits and the forward's alphas) at a row pitch of 8K+4 floats plus label chunks of 12 ints."""
    return 4 * (3 * ((K * K + 3) & ~3) + 32 + NT + nf * 2 * NT * (8 * K + 4) + 2 * NT * 12)


def bwd_route(B, K, nf):
    """The kernel a CRF loss backward staging nf float tensors (2: ner_crf_loglik_bwd, 3: ner_crf_partial_loglik_bwd)
    runs for B sequences of K tags: lane per tag up to NER_CRF_SMALL_B, else thread per sequence with 64-thread CTAs
    above 128 sequences per SM when their shared memory fits, and 32-thread CTAs otherwise."""
    if B <= SMALL_B:
        return "lanes"
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return "nt64" if B > 128 * sms and bwd_smem_bytes(K, 64, nf) <= 227 * 1024 else "nt32"


def crf_grad_ref(x, tags, lens, trans, g=None):
    """x [B,L,K], tags [B,L], lens [B], trans [K,K], g [B] (None: all ones).

    alpha [B,L,K] is the forward recursion (meaningful at t < len), logz [B], d_logits [B,L,K], d_trans [K,K], and
    trans_scale [K,K] = S_ij = sum_b |g_b| sum_t (1[gold pair (i,j) at t] + P(y_{t-1}=i, y_t=j)), the size of what
    d_trans[i][j] sums, against which its error is judged."""
    dev = x.device
    x = x.to(torch.float64)
    tr = trans.to(device=dev, dtype=torch.float64)
    B, L, K = x.shape
    n = lens.to(device=dev, dtype=torch.long).clamp(0, L)
    y = tags.to(device=dev, dtype=torch.long).clamp(0, K - 1)
    g = torch.ones(B, dtype=torch.float64, device=dev) if g is None else g.to(device=dev, dtype=torch.float64)
    steps = torch.arange(L, device=dev)
    valid = steps[None, :] < n[:, None]                                         # [B, L]

    alpha = torch.empty_like(x)
    alpha[:, 0] = x[:, 0]
    for t in range(1, L):
        alpha[:, t] = x[:, t] + torch.logsumexp(alpha[:, t - 1, :, None] + tr[None], dim=1)
    last = alpha[torch.arange(B, device=dev), (n - 1).clamp(min=0)]
    logz = torch.where(n > 0, torch.logsumexp(last, dim=1), torch.zeros((), dtype=torch.float64, device=dev))

    # beta_t = 0 at t >= len-1; u_t = x_t + beta_t feeds the pair marginal of (t-1, t) and beta_{t-1}
    beta = torch.zeros_like(x)
    for t in range(L - 2, -1, -1):
        rec = torch.logsumexp(tr[None] + (x[:, t + 1] + beta[:, t + 1])[:, None, :], dim=2)
        beta[:, t] = torch.where((t < n - 1)[:, None], rec, torch.zeros_like(rec))

    gv = g[:, None] * valid                                                     # g_b at valid steps, else 0
    p = torch.exp(alpha + beta - logz[:, None, None])
    onehot = torch.nn.functional.one_hot(y, K).to(torch.float64)
    d_logits = torch.where(valid[:, :, None], gv[:, :, None] * (onehot - p), torch.zeros_like(x))

    d_trans = torch.zeros((K, K), dtype=torch.float64, device=dev)
    scale = torch.zeros((K, K), dtype=torch.float64, device=dev)
    ga = g.abs()
    for t in range(1, L):
        if not bool(valid[:, t].any()):
            continue
        w = gv[:, t]
        pair = torch.exp(alpha[:, t - 1, :, None] + tr[None] + (x[:, t] + beta[:, t])[:, None, :]
                         - logz[:, None, None])
        pair = torch.where(valid[:, t, None, None], pair, torch.zeros_like(pair))
        d_trans -= torch.einsum("b,bij->ij", w, pair)
        scale += torch.einsum("b,bij->ij", ga, pair)
        d_trans.index_put_((y[:, t - 1], y[:, t]), w, accumulate=True)
        scale.index_put_((y[:, t - 1], y[:, t]), ga * valid[:, t], accumulate=True)
    return CrfGrad(alpha, logz, d_logits, d_trans, g, n, scale)


def row_unit(ref):
    """u_b = |g_b| EPS32 (1 + |log Z_b| + max_{t<len_b, j} |alpha_b,t,j|) sqrt(len_b): the scale of float32 rounding in
    row b's marginals (beta_t is at most |log Z| + |alpha_t| in size)."""
    B, L, _ = ref.alpha.shape
    valid = (torch.arange(L, device=ref.alpha.device)[None, :] < ref.lens[:, None])[:, :, None]
    a = torch.where(valid & torch.isfinite(ref.alpha), ref.alpha.abs(), torch.zeros_like(ref.alpha))
    amax = a.reshape(B, -1).max(dim=1).values
    return ref.g.abs() * EPS32 * (1 + ref.logz.abs() + amax) * ref.lens.clamp(min=1).double().sqrt()


def grad_errors(d_logits, d_trans, ref, rtol):
    """Worst errors of a kernel's (d_logits, d_trans) against `ref` (a CrfGrad):
    (max_b,t,j (|d - ref| - rtol*|ref|) / u_b,  max_ij |d_trans - ref| / S_ij,  max_b,t,j |d - ref| / |g_b|).
    A nonzero error where the scale is 0 (a row with g_b = 0, a transition no path takes) is reported as inf."""
    dl = d_logits.to(device=ref.d_logits.device, dtype=torch.float64)
    dt = d_trans.to(device=ref.d_trans.device, dtype=torch.float64)
    err = (dl - ref.d_logits).abs()
    excess = (err - rtol * ref.d_logits.abs()).clamp(min=0)
    e_dl = _worst_ratio(excess, row_unit(ref)[:, None, None].expand_as(dl))
    e_dt = _worst_ratio((dt - ref.d_trans).abs(), ref.trans_scale)
    return e_dl, e_dt, _worst_ratio(err, ref.g.abs()[:, None, None].expand_as(dl))


def _worst_ratio(err, scale):
    if not bool(torch.isfinite(err).all()):
        return float("inf")
    pos = scale > 0
    if bool((err[~pos] != 0).any()):
        return float("inf")
    return float((err[pos] / scale[pos]).max()) if bool(pos.any()) else 0.0


def assert_grads_close(d_logits, d_trans, ref, rtol, c_dl, tol_s):
    """|d_logits - ref| <= rtol*|ref| + c_dl*u_b elementwise (row_unit), and |d_trans - ref| <= tol_s * S elementwise."""
    e_dl, e_dt, e_g = grad_errors(d_logits, d_trans, ref, rtol)
    assert e_dl <= c_dl, f"d_logits error {e_dl:.3g} u_b ({e_g:.3e} |g_b|) exceeds {c_dl:.3g} u_b"
    assert e_dt <= tol_s, f"d_trans error {e_dt:.3e} S exceeds {tol_s:.1e} S"
    return e_dl, e_dt, e_g
