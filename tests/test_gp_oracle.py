"""The float64 GlobalPointer restatement (tests/_gp_oracle.py) checked on the CPU: the loss against a loop over every span,
its dS against autograd, the gradients of q and k through RoPE against autograd, and RoPE as an orthogonal map whose
scores depend only on j - i."""
import numpy as np
import torch

import _gp_oracle as gp

D = gp.D


def _case(B=3, T=2, L=9, seed=0):
    rng = np.random.default_rng(seed)
    S = torch.from_numpy(rng.normal(scale=2.0, size=(B, T, L, L)))
    lens = np.array([L, 5, 2][:B], np.int32)
    tags = rng.choice([0, 1, 2, 3, 4], size=(B, L)).astype(np.int32)      # O, B-X0, I-X0, B-X1, I-X1
    span_end = gp.targets(tags, lens, [[1, 2], [3, 4]][:T])
    return S, lens, span_end


def test_targets_by_hand():
    tags = np.array([[9, 1, 2, 2, 0, 2, 1, 3, 4, 1]], np.int32)          # I-run without B at 5; B at 6 with no I
    se = gp.targets(tags, [9], [[1, 2], [3, 4]])
    assert se[0, 0].tolist() == [-1, 3, -1, -1, -1, -1, 6, -1, -1, -1]     # position 9 is past seq_len
    assert se[0, 1].tolist() == [-1, -1, -1, -1, -1, -1, -1, 8, -1, -1]


def test_loss_against_a_loop_over_spans():
    S, lens, span_end = _case()
    B, T, L, _ = S.shape
    total = 0.0
    for b in range(B):
        m = min(int(lens[b]), L) - 2
        for t in range(T):
            neg, pos = [0.0], [0.0]
            for i in range(1, m + 1):
                for j in range(i, m + 1):
                    s = float(S[b, t, i, j])
                    (pos if span_end[b, t, i] == j else neg).append(s if span_end[b, t, i] != j else -s)
            total += np.log(np.sum(np.exp(neg))) + np.log(np.sum(np.exp(pos)))
    assert abs(float(gp.loss(S, span_end, lens)) - total / (B * T)) < 1e-12
    assert float(gp.loss(S, np.full_like(span_end, -1), np.zeros(B, np.int32))) == 0.0     # no candidates: 0


def test_d_scores_is_the_autograd_gradient():
    S, lens, span_end = _case(seed=1)
    leaf = S.clone().requires_grad_(True)
    (0.7 * gp.loss(leaf, span_end, lens)).backward()
    assert torch.allclose(gp.d_scores(S, span_end, lens, 0.7), leaf.grad, rtol=0, atol=1e-14)


def test_operand_gradients_through_rope():
    rng = np.random.default_rng(2)
    B, L, T = 2, 7, 2
    q = torch.from_numpy(rng.normal(size=(B, L, T, D))).requires_grad_(True)
    k = torch.from_numpy(rng.normal(size=(B, L, T, D))).requires_grad_(True)
    lens = np.array([7, 4], np.int32)
    span_end = gp.targets(rng.choice([0, 1, 2, 3, 4], size=(B, L)), lens, [[1, 2], [3, 4]])
    qr, kr = gp.operands(q, k)
    S = gp.scores(qr, kr)
    gp.loss(S, span_end, lens).backward()
    dS = gp.d_scores(S.detach(), span_end, lens)
    dqr = torch.einsum('btij,bjtd->bitd', dS, kr.detach())                  # dQ' = dS K'
    dkr = torch.einsum('btij,bitd->bjtd', dS, qr.detach())                  # dK' = dS^T Q'
    pos = np.arange(L)
    back = lambda x: gp.rope(x, -pos)                                       # R^T = rotation by the negative angle
    assert torch.allclose(back(dqr) / np.sqrt(D), q.grad, atol=1e-12)
    assert torch.allclose(back(dkr), k.grad, atol=1e-12)


def test_rope_is_orthogonal_and_relative():
    rng = np.random.default_rng(3)
    L = 40
    x = torch.from_numpy(rng.normal(size=(1, L, D)))
    r = gp.rope(x, np.arange(L))
    assert torch.allclose(r.norm(dim=-1), x.norm(dim=-1), atol=1e-12)
    assert torch.allclose(gp.rope(r, -np.arange(L)), x, atol=1e-12)
    qv, kv = torch.from_numpy(rng.normal(size=D)), torch.from_numpy(rng.normal(size=D))
    q = qv.expand(1, L, 1, D).clone()
    k = kv.expand(1, L, 1, D).clone()
    S = gp.scores(*gp.operands(q, k))[0, 0]
    for d in range(-5, 6):
        diag = torch.diagonal(S, offset=d)
        assert torch.allclose(diag, diag[0].expand_as(diag), atol=1e-12)
    assert not torch.allclose(torch.diagonal(S, 1)[0], torch.diagonal(S, 2)[0])


def test_decode_by_hand():
    L, T = 8, 2
    S = np.full((1, T, L, L), -1.0, np.float32)
    S[0, 0, 1, 4], S[0, 1, 2, 3], S[0, 1, 1, 4] = 2.0, 3.0, 0.5                # nested, and a start with two types
    pred, words, probs, counts = gp.decode(S, [7], [[2, 3], [4, 5]], 1, 8, 9, 2)
    assert counts.tolist() == [3]
    assert words.tolist() == [[1 | 5 << 12, 1 | 5 << 12 | 1 << 24]]
    assert pred.tolist() == [[8, 1, 4, 5, 1, 1, 9, 0]]                      # the best span (2, 3) wins; (1, 4) overlaps it
