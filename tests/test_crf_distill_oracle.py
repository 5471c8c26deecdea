"""CPU: the float64 distillation reference (tests/_crf_distill_oracle.py) against a sum over every path, and its
gradient against central finite differences of that sum."""
import numpy as np
import pytest
import torch

from _crf_distill_oracle import brute_kl, distill_ref


def _row(n, K, seed, wide=False, inf=False):
    rng = np.random.default_rng(seed)
    xt, xs = rng.normal(size=(n, K)) * 2, rng.normal(size=(n, K)) * 2
    sd = 6.0 if wide else 0.7
    trt, trs = rng.normal(size=(K, K)) * sd, rng.normal(size=(K, K)) * sd
    if inf and K > 1:
        trt[0, 1] = trt[1, 0] = -np.inf
    return xt, trt, xs, trs


def _ref(xt, trt, xs, trs, n, L, tau):
    K = xs.shape[1]
    pad = lambda x: torch.from_numpy(np.concatenate([x, np.zeros((L - n, K))])[None])     # noqa: E731
    return distill_ref(pad(xt), torch.from_numpy(trt), pad(xs), torch.from_numpy(trs), torch.tensor([n]), tau)


CASES = [(1, 1), (1, 5), (2, 3), (3, 4), (5, 3), (4, 10), (6, 6), (2, 32), (10, 3)]    # (n, K): K^n <= 1e5


@pytest.mark.parametrize("tau", [0.5, 1.0, 2.0])
@pytest.mark.parametrize("n,K", CASES)
@pytest.mark.parametrize("kind", ["narrow", "wide", "inf"])
def test_kl_equals_the_sum_over_every_path(n, K, tau, kind):
    xt, trt, xs, trs = _row(n, K, seed=n * 100 + K, wide=kind == "wide", inf=kind == "inf")
    ref = _ref(xt, trt, xs, trs, n, n + 2, tau)
    want = brute_kl(xt, trt, xs, trs, tau)
    assert want >= -1e-12
    assert abs(float(ref.kl[0]) - want) <= 1e-9 * max(1.0, abs(want))


@pytest.mark.parametrize("tau", [0.5, 1.0, 2.0])
@pytest.mark.parametrize("n,K", [(1, 3), (3, 4), (4, 3), (5, 2)])
def test_gradient_matches_central_differences(n, K, tau):
    xt, trt, xs, trs = _row(n, K, seed=7 * n + K)
    ref = _ref(xt, trt, xs, trs, n, n, tau)
    h = 1e-5
    for idx in np.ndindex(xs.shape):
        xp, xm = xs.copy(), xs.copy()
        xp[idx] += h
        xm[idx] -= h
        fd = (brute_kl(xt, trt, xp, trs, tau) - brute_kl(xt, trt, xm, trs, tau)) / (2 * h)
        assert abs(float(ref.grad.d_logits[0][idx]) - fd) < 1e-6, idx
    for idx in np.ndindex(trs.shape):
        tp, tm = trs.copy(), trs.copy()
        tp[idx] += h
        tm[idx] -= h
        fd = (brute_kl(xt, trt, xs, tp, tau) - brute_kl(xt, trt, xs, tm, tau)) / (2 * h)
        assert abs(float(ref.grad.d_trans[idx]) - fd) < 1e-6, idx


def test_equal_models_and_empty_rows_give_zero():
    xt, trt, _, _ = _row(4, 5, seed=3)
    ref = _ref(xt, trt, xt, trt, 4, 6, 1.0)
    assert abs(float(ref.kl[0])) < 1e-12 and float(ref.grad.d_logits.abs().max()) < 1e-12
    x = torch.randn(3, 4, 5, dtype=torch.float64)
    r = distill_ref(x, torch.randn(5, 5), x * 2, torch.randn(5, 5), torch.tensor([0, -2, 0]))
    assert (r.kl == 0).all() and (r.grad.d_logits == 0).all() and (r.grad.d_trans == 0).all()
