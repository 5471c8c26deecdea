"""CPU: the numpy restatement of the masking rule against hand-worked rows, the budget against Google's expression, and the
float64 head and loss against torch's cross-entropy."""
import numpy as np
import pytest
import torch

import _mlm_oracle as mo
from chinesener_b200 import mlm


def test_hash3_matches_the_device_formula_on_known_values():
    # common.cuh hash3, worked by hand with Python integers
    def ref(a, b, c):
        m = 0xFFFFFFFF
        x = (a * 0x9E3779B1 & m) ^ ((b + 0x7F4A7C15 & m) * 0x85EBCA77 & m) ^ ((c + 0x165667B1 & m) * 0xC2B2AE3D & m)
        x ^= x >> 16
        x = x * 0x7FEB352D & m
        x ^= x >> 15
        x = x * 0x846CA68B & m
        return x ^ (x >> 16)
    for a, b, c in [(0, 0, 0), (1, 2, 3), (0xFFFFFFFF, 0xFFFFFFFF, 511), (12345, 678, 9)]:
        assert int(mo.hash3(a, b, c)) == ref(a, b, c)


@pytest.mark.parametrize("n", [0, 1, 2, 3])
def test_short_rows(n):
    toks = np.arange(10, 18)
    row, chosen = mo.mask_row(toks, n, None, mo.google_budget(n, 0.15, 20), 5, 0, 100, 3)
    assert chosen == ([1] if n == 3 else [])          # n = 3: the only candidate, budget max(1, round(0.45)) = 1
    assert (row[[i for i in range(8) if i not in chosen]] == toks[[i for i in range(8) if i not in chosen]]).all()


def test_whole_words_that_do_not_fit_are_skipped():
    # n = 8: candidates 1..6, words [1, 2, 3] and [4] and [5, 6]
    ws = np.array([0, 1, 0, 0, 1, 1, 0, 0], np.uint8)
    assert mo.words_of_row(8, ws) == [(1, 3), (4, 1), (5, 2)]
    for seed in range(20):
        _, chosen = mo.mask_row(np.arange(8), 8, ws, 1, seed, 0, 100, 3)
        assert chosen == [4]                           # the only word of length <= 1, whatever the order
        _, chosen = mo.mask_row(np.arange(8), 8, ws, 2, seed, 0, 100, 3)
        assert chosen in ([4], [5, 6])                 # the first of them in key order; the other no longer fits
        _, chosen = mo.mask_row(np.arange(8), 8, ws, 6, seed, 0, 100, 3)
        assert chosen == [1, 2, 3, 4, 5, 6]


def test_all_one_word_rows():
    ws = np.zeros(8, np.uint8)                         # position 1 starts the only word: 1..n-2
    for n in (4, 8):
        assert mo.words_of_row(n, ws) == [(1, n - 2)]
        assert mo.mask_row(np.arange(8), n, ws, n - 3, 1, 0, 100, 3)[1] == []
        assert mo.mask_row(np.arange(8), n, ws, n - 2, 1, 0, 100, 3)[1] == list(range(1, n - 1))


def test_unused_slots_point_at_cls_with_label_minus_one():
    toks = np.arange(10, 26).reshape(2, 8)
    ws = np.array([[0, 1, 0, 0, 0, 0, 0, 0]] * 2, np.uint8)       # one word of 6 tokens per row
    offsets = np.array([0, 2, 4], np.int32)
    masked, pos, lab = mo.mlm_mask(toks, np.array([8, 8]), ws, offsets, 3, 100, 3)
    assert pos.tolist() == [0, 0, 8, 8] and lab.tolist() == [-1] * 4 and (masked == toks).all()


def test_corruption_split_and_random_ids():
    seed, V = 99, 1000
    u = np.array([int(mo.mask_hash(seed, 1, 0, t)) >> 8 for t in range(20000)]) / 2 ** 24
    assert 0.79 < (u < 0.8).mean() < 0.81 and 0.09 < ((u >= 0.8) & (u < 0.9)).mean() < 0.11
    ids = [(int(mo.mask_hash(seed, 2, 0, t)) * V) >> 32 for t in range(2000)]
    assert min(ids) >= 0 and max(ids) < V and len(set(ids)) > 800


def test_budget_matches_googles_expression_at_half_way_lengths():
    # n * 0.1 = x.5 at n = 5, 15, 25, 35: Python 3 rounds half to even
    for p in (0.1, 0.15, 0.5, 1.0):
        for n in range(0, 80):
            assert mlm.prediction_budget([n], p, 20)[0] == mo.google_budget(n, p, 20), (n, p)
    assert mlm.prediction_budget([5, 15, 25, 35], 0.1, 20).tolist() == [1, 2, 2, 4]   # round(0.5)=0 -> max(1, .); 1.5 -> 2
    assert mlm.pred_offsets(np.array([2, 0, 3])).tolist() == [0, 2, 2, 5]


def test_float64_xent_matches_torch_cross_entropy():
    rng = np.random.default_rng(0)
    M, V, ld = 9, 37, 40
    z = rng.normal(0, 3, (M, ld))
    y = rng.integers(0, V, M)
    y[[1, 4]] = -1
    loss, count, correct, pred, d = mo.vocab_xent(z, y, V, d_loss=2.0)
    zt = torch.tensor(z[:, :V], requires_grad=True)
    yt = torch.tensor(y)
    ref = torch.nn.functional.cross_entropy(zt, yt, ignore_index=-1)
    (2.0 * ref).backward()
    assert count == 7 and abs(loss - float(ref.detach())) < 1e-12
    assert np.allclose(d[:, :V], zt.grad.numpy(), atol=1e-14) and (d[:, V:] == 0).all() and (d[[1, 4]] == 0).all()
    assert correct == int(((pred == y) & (y >= 0)).sum())


def test_float64_head_matches_torch_cross_entropy():
    torch.manual_seed(0)
    H, V, M = 16, 30, 6
    w = {"cls/predictions/transform/dense/kernel": torch.randn(H, H) * 0.2, "cls/predictions/transform/dense/bias": torch.randn(H),
         "cls/predictions/transform/LayerNorm/gamma": torch.rand(H) + 0.5, "cls/predictions/transform/LayerNorm/beta": torch.randn(H),
         "bert/embeddings/word_embeddings": torch.randn(V, H), "cls/predictions/output_bias": torch.randn(V)}
    h = torch.randn(M, H, dtype=torch.float64)
    y = torch.tensor([3, -1, 0, 29, -1, 7])
    logits = mo.head_logits(h, w, V)
    ref = torch.nn.functional.cross_entropy(logits, y, ignore_index=-1)
    assert abs(float(mo.masked_lm_loss(logits, y)) - float(ref)) < 1e-12
    t = torch.nn.functional.layer_norm(torch.nn.functional.gelu(h @ w["cls/predictions/transform/dense/kernel"].double()
                                                                + w["cls/predictions/transform/dense/bias"].double(), approximate="tanh"),
                                       (H,), w["cls/predictions/transform/LayerNorm/gamma"].double(),
                                       w["cls/predictions/transform/LayerNorm/beta"].double(), eps=1e-12)
    assert torch.allclose(logits, t @ w["bert/embeddings/word_embeddings"].double().T + w["cls/predictions/output_bias"].double(),
                          atol=1e-12)
