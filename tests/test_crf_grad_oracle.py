"""CPU: the batched float64 CRF forward-backward (tests/_crf_grad_oracle.py) against the per-sequence numpy oracle and
autograd of the torch restatement, and the gradient comparator against plausible wrong answers."""
import numpy as np
import pytest
import torch

from oracle import crf, crf_torch

from _crf_grad_oracle import TOL, assert_grads_close, crf_grad_ref, grad_errors


def _case(B, L, K, seed, forbid=False):
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(B, L, K, generator=gen, dtype=torch.float64) * 2
    tr = torch.randn(K, K, generator=gen, dtype=torch.float64)
    lens = torch.randint(0, L + 1, (B,), generator=gen, dtype=torch.int32)
    tags = torch.randint(0, K, (B, L), generator=gen, dtype=torch.int32)
    lens[0] = L
    if B > 2:
        lens[1], lens[2] = 1, 0
    if forbid and K > 1:
        tr[0, 1] = -float("inf")
        tags[tags == 0] = 1                          # the gold path never takes the forbidden edge
    return x, tags, lens, tr


@pytest.mark.parametrize("B,L,K,forbid", [(9, 13, 5, False), (6, 1, 4, False), (5, 7, 1, False), (7, 11, 6, True),
                                          (4, 9, 2, True), (12, 20, 10, False)])
def test_reference_matches_per_sequence_forward_backward(B, L, K, forbid):
    x, tags, lens, tr = _case(B, L, K, seed=B * 100 + L + K, forbid=forbid)
    ref = crf_grad_ref(x, tags, lens, tr)
    dx, dtr = crf.crf_marginal_grads(x.numpy(), tags.numpy(), lens.numpy(), tr.numpy())
    np.testing.assert_allclose(ref.d_logits.numpy(), dx, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(ref.d_trans.numpy(), dtr, rtol=1e-12, atol=1e-12)
    logz, alphas = crf.crf_log_norm(x.numpy(), lens.numpy(), tr.numpy(), return_alphas=True)
    np.testing.assert_allclose(ref.logz.numpy(), logz, rtol=1e-12, atol=1e-12)
    for b in range(B):
        n = int(lens[b])
        np.testing.assert_allclose(ref.alpha[b, :n].numpy(), alphas[b, :n], rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("B,L,K,forbid", [(9, 13, 5, False), (6, 1, 4, False), (5, 7, 1, False), (7, 11, 6, True),
                                          (12, 20, 10, False)])
def test_reference_matches_weighted_autograd(B, L, K, forbid):
    x, tags, lens, tr = _case(B, L, K, seed=B * 7 + L + K, forbid=forbid)
    g = torch.empty(B, dtype=torch.float64).uniform_(-2, 2, generator=torch.Generator().manual_seed(B))
    g[::4] = 0
    xl, trl = x.clone().requires_grad_(True), tr.clone().requires_grad_(True)
    ll = crf_torch.crf_log_likelihood(xl, tags, lens, trl)
    (ll * g).sum().backward()
    ref = crf_grad_ref(x, tags, lens, tr, g)
    torch.testing.assert_close(ref.d_logits, xl.grad, rtol=1e-12, atol=1e-12)
    d_trans = trl.grad if trl.grad is not None else torch.zeros_like(tr)   # L = 1: no transition is scored
    torch.testing.assert_close(ref.d_trans, d_trans, rtol=1e-12, atol=1e-12)


def test_reference_conventions():
    """Lengths are clamped to [0, L], tags to [0, K-1]; a length <= 0 has log Z = 0 and no gradient."""
    B, L, K = 6, 8, 5
    x, tags, lens, tr = _case(B, L, K, seed=3)
    lens_raw = lens.clone()
    lens_raw[3], lens_raw[4] = L + 9, -4
    tags_raw = tags.clone()
    tags_raw[5, ::2] = K + 3
    tags_raw[5, 1::2] = -2
    got = crf_grad_ref(x, tags_raw, lens_raw, tr)
    want = crf_grad_ref(x, tags_raw.clamp(0, K - 1), lens_raw.clamp(0, L), tr)
    torch.testing.assert_close(got.d_logits, want.d_logits, rtol=0, atol=0)
    torch.testing.assert_close(got.d_trans, want.d_trans, rtol=0, atol=0)
    assert got.logz[4] == 0 and (got.d_logits[4] == 0).all() and got.lens[3] == L


def _mutations(x, tags, lens, tr, g, ref, nt):
    """Wrong answers a broken kernel could plausibly give, each derived from the reference."""
    B, L, K = x.shape
    out = {}
    g_drop = g.clone()
    g_drop[nt:2 * nt] = 0                                         # the second CTA's rows never reach the output
    r = crf_grad_ref(x, tags, lens, tr, g_drop)
    out["cta_dropped"] = (r.d_logits, r.d_trans)
    # unary marginal of step t-1 used at step t:  g (onehot_t - P_{t-1}) = dl_{t-1} + g (onehot_t - onehot_{t-1})
    oh = torch.nn.functional.one_hot(tags.long().clamp(0, K - 1), K).to(torch.float64)
    valid = (torch.arange(L)[None, :] < ref.lens[:, None])
    shifted = ref.d_logits.clone()
    shifted[:, 1:] = ref.d_logits[:, :-1] + g[:, None, None] * (oh[:, 1:] - oh[:, :-1])
    out["marginal_shifted"] = (torch.where(valid[:, :, None], shifted, torch.zeros_like(shifted)), ref.d_trans)
    r = crf_grad_ref(x, tags, lens, tr, g.roll(1))
    out["d_ll_rolled"] = (r.d_logits, r.d_trans)
    out["d_trans_transposed"] = (ref.d_logits, ref.d_trans.t().contiguous())
    r = crf_grad_ref(x, tags, lens, tr, torch.full_like(g, 0.75))  # g_b = scale: d_ll ignored
    out["d_ll_ignored"] = (r.d_logits, r.d_trans)
    return out


def test_comparator_rejects_wrong_gradients():
    B, L, K, nt = 101, 19, 7, 32
    x, tags, lens, tr = _case(B, L, K, seed=5)
    gen = torch.Generator().manual_seed(6)
    g = torch.empty(B, dtype=torch.float64).uniform_(-2, 2, generator=gen) * 0.75
    g[::7] = 0
    ref = crf_grad_ref(x, tags, lens, tr, g)
    rtol, c_dl, tol_s = (max(t[i] for t in TOL.values()) for i in range(3))     # the loosest tolerances in use
    # the float32-rounded reference passes
    assert_grads_close(ref.d_logits.float(), ref.d_trans.float(), ref, rtol, c_dl, tol_s)
    for name, (dl, dt) in _mutations(x, tags, lens, tr, g, ref, nt).items():
        e_dl, e_dt, _ = grad_errors(dl.float(), dt.float(), ref, rtol)
        assert e_dl > c_dl or e_dt > tol_s, name
        with pytest.raises(AssertionError):
            assert_grads_close(dl.float(), dt.float(), ref, rtol, c_dl, tol_s)


def test_comparator_demands_exact_zeros_on_masked_rows():
    B, L, K = 9, 6, 4
    x, tags, lens, tr = _case(B, L, K, seed=8)
    g = torch.linspace(-1, 1, B, dtype=torch.float64)
    g[4] = 0
    ref = crf_grad_ref(x, tags, lens, tr, g)
    dl = ref.d_logits.clone()
    dl[4, 0, 0] = 1e-30                                          # a masked row must be exactly zero
    assert grad_errors(dl, ref.d_trans, ref, 0.0)[0] == float("inf")
