"""The bert_mrc_span restatement (tests/_mrc_span_oracle.py) pinned without a GPU: hand-worked targets, the match head and
its loss against float64 autograd on the explicit [P, L, L, I] tensor (and the closed-form backward the kernels use), and
the projection's tie rules."""
import numpy as np
import pytest
import torch

import _mrc_span_oracle as so


def _targets(labels, n):
    start, end, span_end = so.targets(np.array([labels], np.int32), [n])
    return start[0].tolist(), end[0].tolist(), span_end[0].tolist()


def test_targets_hand_worked():
    # [CLS] B I I O I I B B I [SEP]: spans 1..3, 7..7, 8..9; the I-run 5..6 has no B in front
    start, end, span_end = _targets([0, 1, 2, 2, 0, 2, 2, 1, 1, 2, 0], 11)
    assert start == [0, 1, 0, 0, 0, 0, 0, 1, 1, 0, 0]
    assert end == [0, 0, 0, 1, 0, 0, 0, 1, 0, 1, 0]
    assert span_end == [-1, 3, -1, -1, -1, -1, -1, 7, 9, -1, -1]
    # adjacent spans B B I: 1..1 and 2..3
    assert _targets([0, 1, 1, 2, 0], 5) == ([0, 1, 1, 0, 0], [0, 1, 0, 1, 0], [-1, 1, 3, -1, -1])
    # a span ending at len - 2, then padding that would extend it
    assert _targets([0, 0, 1, 2, 0, 2, 2], 5) == ([0, 0, 1, 0, 0, 0, 0], [0, 0, 0, 1, 0, 0, 0], [-1, -1, 3, -1, -1, -1, -1])


@pytest.mark.parametrize("n", [0, 1, 2, 3])
def test_targets_short_sentences(n):
    labels = [1, 2, 1, 2, 2, 1]
    start, end, span_end = _targets(labels, n)
    ref_start = [int(s < n and labels[s] == 1) for s in range(6)]
    assert start == ref_start
    assert all(e == 0 for e in end[n:]) and all(r == -1 for r in span_end[n:])
    assert all(r < n for r in span_end)
    assert so.candidates([n], 6).sum() == max(n - 2, 0) * max(n - 1, 0) // 2


def _case(P, L, I, seed):
    g = torch.Generator().manual_seed(seed)
    U = torch.randn(P, L, I, generator=g, dtype=torch.float64)
    V = torch.randn(P, L, I, generator=g, dtype=torch.float64)
    b1 = 0.5 * torch.randn(I, generator=g, dtype=torch.float64)
    w2 = torch.randn(I, generator=g, dtype=torch.float64) / I ** 0.5
    b2 = torch.tensor(0.1, dtype=torch.float64)
    lens = [L, 0, 3, 4, L - 1][:P]
    labels = np.random.default_rng(seed).integers(0, 3, size=(P, L)).astype(np.int32)
    return U, V, b1, w2, b2, lens, labels


@pytest.mark.parametrize("keep", [1.0, 0.8])
def test_match_head_and_loss_against_explicit_autograd(keep):
    P, L, I, seed = 5, 9, 32, 1234567890123
    U, V, b1, w2, b2, lens, labels = _case(P, L, I, seed=3)
    _, _, span_end = so.targets(labels, lens)
    leaves = [t.clone().requires_grad_(True) for t in (U, V, b1, w2, b2)]
    z = so.match_logits(*leaves, lens, keep=keep, seed=seed, rows=3)
    loss = so.bce_loss(z, span_end, lens)
    loss.backward()
    # the explicit [P, L, L, I] activation tensor
    ref = [t.clone().requires_grad_(True) for t in (U, V, b1, w2, b2)]
    X = ref[0][:, :, None, :] + ref[1][:, None, :, :] + ref[2]
    A = so.gelu_tanh(X)
    if keep < 1.0:
        A = A * torch.stack([so.dropout_scale(seed, p, np.arange(L), np.arange(L), L, I, keep) for p in range(P)])
    zf = A @ ref[3] + ref[4]
    cand = torch.as_tensor(so.candidates(lens, L))
    y = torch.as_tensor(span_end[:, :, None] == np.arange(L)[None, None, :], dtype=torch.float64)
    ref_loss = torch.nn.functional.binary_cross_entropy_with_logits(zf[cand], y[cand])
    ref_loss.backward()
    torch.testing.assert_close(z.detach(), torch.where(cand, zf, torch.zeros_like(zf)).detach(), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(loss.detach(), ref_loss.detach(), rtol=1e-12, atol=1e-12)
    for a, b in zip(leaves, ref):
        torch.testing.assert_close(a.grad, b.grad, rtol=1e-10, atol=1e-12)
    # the closed form the backward kernels evaluate: dz = (sigmoid(z) - y) / N, dx = dz w2 m g'(x)
    with torch.no_grad():
        n = int(cand.sum())
        dz = torch.where(cand, (torch.sigmoid(zf) - y) / n, torch.zeros_like(zf))
        x = X
        t = torch.tanh(so.C0 * (x + 0.044715 * x ** 3))
        gp = 0.5 * (1 + t) + 0.5 * x * (1 - t * t) * so.C0 * (1 + 3 * 0.044715 * x * x)
        m = torch.ones_like(x) if keep == 1.0 else torch.stack(
            [so.dropout_scale(seed, p, np.arange(L), np.arange(L), L, I, keep) for p in range(P)])
        dx = dz[..., None] * w2 * m * gp
        torch.testing.assert_close(dx.sum(2), ref[0].grad)
        torch.testing.assert_close(dx.sum(1), ref[1].grad)
        torch.testing.assert_close(dx.sum((0, 1, 2)), ref[2].grad)
        torch.testing.assert_close((dz[..., None] * m * so.gelu_tanh(x)).sum((0, 1, 2)), ref[3].grad)
        torch.testing.assert_close(dz.sum(), ref[4].grad)


def test_loss_without_candidates_is_zero():
    U, V, b1, w2, b2, _, labels = _case(2, 4, 32, seed=1)
    lens = [2, 0]
    z = so.match_logits(U, V, b1, w2, b2, lens)
    assert float(so.bce_loss(z, so.targets(labels, lens)[2], lens)) == 0.0 and not z.any()


def test_dropout_keeps_about_keep():
    s = so.dropout_scale(99, 3, np.arange(40), np.arange(40), 40, 64, 0.9)
    frac = float((s > 0).double().mean())
    assert abs(frac - 0.9) < 0.01
    assert torch.allclose(s[s > 0], torch.tensor(1 / 0.9, dtype=torch.float64), rtol=1e-6)


TT = [[2, 3], [4, 5], [6, 7]]


def test_projection_tie_rules():
    n, L = 10, 12
    # equal z: the lower type wins, then the lower start, then the lower end
    assert so.project([(2, 3, 1, 1.0), (2, 3, 0, 1.0)], n, TT, 1, 8, 9, L)[2:4].tolist() == [2, 3]
    assert so.project([(3, 4, 0, 1.0), (2, 3, 0, 1.0)], n, TT, 1, 8, 9, L)[1:6].tolist() == [1, 2, 3, 1, 1]
    assert so.project([(2, 4, 0, 1.0), (2, 3, 0, 1.0)], n, TT, 1, 8, 9, L)[1:6].tolist() == [1, 2, 3, 1, 1]
    # a higher z wins regardless of type; a nested span overlapping it is skipped, a disjoint one kept
    tags = so.project([(1, 5, 0, 0.5), (2, 3, 2, 2.0), (6, 8, 1, 0.1)], n, TT, 1, 8, 9, L)
    assert tags.tolist() == [8, 1, 6, 7, 1, 1, 4, 5, 5, 9, 0, 0]


def test_decode_restatement_lists_nested_spans():
    T, L = 2, 8
    sl = np.zeros((T, L, 2), np.float32)
    el = np.zeros((T, L, 2), np.float32)
    sl[0, 1, 1] = el[0, 2, 1] = el[0, 4, 1] = 1.0      # type 0: one start, two ends
    sl[1, 2, 1] = el[1, 3, 1] = 1.0                     # type 1: nested inside
    z = np.full((T, L, L), -1.0, np.float32)
    z[0, 1, 2], z[0, 1, 4], z[1, 2, 3] = 0.5, 2.0, 3.0
    pred, words, probs, counts = so.decode(sl, el, z, [7], [[2, 3], [4, 5]], 1, 8, 9, cap=2)
    assert counts.tolist() == [3]                       # past cap: dropped, still counted
    assert words[0].tolist() == [1 | 3 << 12, 1 | 5 << 12]
    assert probs[0, 1] == so.sigmoid32(2.0)
    assert pred[0].tolist() == [8, 1, 4, 5, 1, 1, 9, 0]  # z = 3 wins; both type-0 spans overlap it
