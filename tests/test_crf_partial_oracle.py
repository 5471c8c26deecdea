"""CPU: the float64 partial-annotation CRF reference (tests/_crf_partial_oracle.py) against brute-force path
enumeration, and every edge case of its definition."""
import numpy as np
import pytest
import torch

from _crf_grad_oracle import crf_grad_ref
from _crf_partial_oracle import allowed_tags, brute_force_partial, partial_grad_ref, step_pair


def _case(B, L, K, seed, forbid=False):
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(B, L, K, generator=gen, dtype=torch.float64) * 2
    tr = torch.randn(K, K, generator=gen, dtype=torch.float64)
    lens = torch.randint(0, L + 1, (B,), generator=gen, dtype=torch.int32)
    lens[0] = L
    if B > 2:
        lens[1], lens[2] = 1, 0
    full = (1 << K) - 1
    mask = torch.randint(1, full + 1, (B, L), generator=gen, dtype=torch.int64)      # random non-empty subsets
    onehot = 1 << torch.randint(0, K, (B, L), generator=gen, dtype=torch.int64)
    pick = torch.randint(0, 3, (B, L), generator=gen)
    mask = torch.where(pick == 0, onehot, torch.where(pick == 1, torch.full_like(mask, full), mask))
    if forbid and K > 1:
        tr[0, 1] = -float("inf")
    return x, mask.to(torch.int32), lens, tr


@pytest.mark.parametrize("B,L,K,forbid", [(6, 5, 3, False), (5, 4, 4, False), (4, 5, 2, True), (5, 3, 1, False),
                                          (4, 1, 4, False), (5, 4, 3, True)])
def test_reference_matches_brute_force(B, L, K, forbid):
    x, mask, lens, tr = _case(B, L, K, seed=B * 100 + L * 10 + K, forbid=forbid)
    g = torch.linspace(-1.5, 0.5, B, dtype=torch.float64)
    ref = partial_grad_ref(x, mask, lens, tr, g)
    allowed = allowed_tags(mask, K).numpy()
    pair_sum = np.zeros((K, K))
    for b in range(B):
        n = int(lens[b])
        ll, unary, pair = brute_force_partial(x[b].numpy(), allowed[b], tr.numpy(), n)
        np.testing.assert_allclose(float(ref.ll[b]), ll, rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(ref.grad.d_logits[b, :n].numpy(), float(g[b]) * unary, rtol=1e-10, atol=1e-12)
        assert (ref.grad.d_logits[b, n:] == 0).all()
        pair_sum += float(g[b]) * pair
    np.testing.assert_allclose(ref.grad.d_trans.numpy(), pair_sum, rtol=1e-10, atol=1e-12)


def test_one_hot_mask_is_the_ordinary_crf():
    x, _, lens, tr = _case(7, 6, 4, seed=3)
    tags = torch.randint(0, 4, (7, 6), generator=torch.Generator().manual_seed(4), dtype=torch.int32)
    g = torch.full((7,), -1.0 / 7, dtype=torch.float64)
    ref = partial_grad_ref(x, (1 << tags.long()).to(torch.int32), lens, tr, g)
    full = crf_grad_ref(x, tags, lens, tr, g)
    gold = torch.stack([x[b, torch.arange(6), tags[b].long()][:int(lens[b])].sum()
                        + tr[tags[b, :-1].long(), tags[b, 1:].long()][:max(int(lens[b]) - 1, 0)].sum() for b in range(7)])
    torch.testing.assert_close(ref.ll, torch.where(lens > 0, gold - full.logz, torch.zeros_like(gold)), rtol=1e-12,
                               atol=1e-12)
    torch.testing.assert_close(ref.grad.d_logits, full.d_logits, rtol=1e-10, atol=1e-12)
    torch.testing.assert_close(ref.grad.d_trans, full.d_trans, rtol=1e-10, atol=1e-12)


def test_edge_cases():
    B, L, K = 5, 4, 3
    x, _, lens, tr = _case(B, L, K, seed=11)
    lens = torch.tensor([4, 0, 3, 4, 2], dtype=torch.int32)
    mask = torch.full((B, L), (1 << K) - 1, dtype=torch.int32)
    mask[2, 1] = 0                       # empty set inside the row: -inf, no gradient
    mask[4, 3] = 0                       # empty set past seq_len: ignored
    mask[3] |= -(1 << 31) | (1 << K)     # bits >= K: ignored
    ref = partial_grad_ref(x, mask, lens, tr)
    assert float(ref.ll[0]) == pytest.approx(0, abs=1e-12) and float(ref.ll[1]) == 0.0
    assert float(ref.ll[2]) == -float("inf") and bool(ref.empty[2]) and not bool(ref.empty[4])
    assert abs(float(ref.ll[3])) < 1e-12 and abs(float(ref.ll[4])) < 1e-12
    assert ref.grad.d_logits.abs().max() < 1e-12          # all-allowed rows, the empty row, the empty sequence
    assert ref.grad.d_trans.abs().max() < 1e-12


def test_allowed_tags_reads_bit_31_and_ignores_bits_past_k():
    m = torch.tensor([[-(1 << 31) | 5, 1 << 3]], dtype=torch.int32)
    a = allowed_tags(m, 32)
    assert a[0, 0].nonzero().flatten().tolist() == [0, 2, 31]
    assert allowed_tags(m, 3)[0, 1].tolist() == [False, False, False]


C_T = 4.0   # d_trans bound of tests/test_crf_partial_gpu.py: tol_s S + C_T U


@pytest.mark.parametrize("trans,t", [("fast", 8), ("fast", 9), ("wide", 64), ("fast", 127)])
def test_d_trans_bound_catches_a_skipped_step(trans, t):
    """At L = 128 the d_trans bound of the GPU tests rejects a kernel that drops the pair marginal of one step (a chunk
    or group boundary, the middle, the last step), on every route: the share of one step is ~S/127, the bound
    2e-5 S + C_T U with U the float32 rounding of log-domain marginals (here U <= 5e-4 S)."""
    gen = torch.Generator().manual_seed(t)
    B, L, K = 64, 128, 10
    x = torch.randn(B, L, K, generator=gen, dtype=torch.float64) * 2
    tr = torch.randn(K, K, generator=gen, dtype=torch.float64) * (12 if trans == "wide" else 0.5)
    lens = torch.full((B,), L, dtype=torch.int32)
    onehot = 1 << torch.randint(0, K, (B, L), generator=gen, dtype=torch.int64)
    mask = torch.where(torch.rand(B, L, generator=gen) < 0.3, torch.full_like(onehot, (1 << K) - 1), onehot)
    mask = mask.to(torch.int32)
    g = torch.randn(B, generator=gen, dtype=torch.float64) * 0.75
    ref = partial_grad_ref(x, mask, lens, tr, g)
    wrong = ref.grad.d_trans - step_pair(x, mask, tr, g, t)
    excess = ((wrong - ref.grad.d_trans).abs() - 2e-5 * ref.grad.trans_scale).clamp(min=0)
    pos = ref.trans_unit > 0
    assert float((excess[pos] / ref.trans_unit[pos]).max()) > 4 * C_T
