"""GPU: the wgmma attention kernel (csrc/attention_tc.cu), one warpgroup per (sequence, head, 64-query-row tile), at the
edges of its grid: lengths on both sides of a tile boundary mixed in one batch, batches of thousands of tiles (many
waves of CTAs per SM), padded mode, and sequences that must not see their neighbours.  ctx is always written over NaN,
so that a row the kernel skips shows up."""
import math

import numpy as np
import pytest
import torch

from chinesener_b200 import _lib, synthetic
from test_attention_tc_gpu import _ref_packed

pytestmark = pytest.mark.gpu
D = 64
EDGE_LENS = [1, 63, 64, 65, 127, 128, 129, 255, 256]


def _attend(qkv, NH, lens=None, mask=None, B=None, L=None):
    """ner_bert_attention (inference) into a ctx pre-filled with NaN; packed mode from `lens`, padded mode from `mask`."""
    ctx = torch.full((qkv.shape[0], NH * D), float("nan"), dtype=torch.bfloat16, device="cuda")
    cu = None
    if lens is not None:
        B, L = len(lens), max(lens)
        cu = torch.tensor([0] + list(np.cumsum(lens)), dtype=torch.int32, device="cuda")
    _lib.check(_lib.lib().ner_bert_attention(_lib.ptr(qkv), _lib.ptr(mask), _lib.ptr(ctx), B, L, NH, D, 1.0 / math.sqrt(D),
                                             -10000.0, _lib.ptr(cu), int(qkv.shape[0]), 1.0, 0, _lib.stream()))
    return ctx


def _qkv(T, NH, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(T, 3 * NH * D, generator=g).to(torch.bfloat16).cuda()


@pytest.mark.parametrize("NH", [1, 3, 12])
def test_tile_edge_lengths_mixed_in_one_batch(NH):
    lens = [int(n) for n in np.random.default_rng(NH).permutation(EDGE_LENS * 2)]
    qkv = _qkv(sum(lens), NH, seed=NH)
    out = _attend(qkv, NH, lens)
    assert torch.isfinite(out.float()).all()
    torch.testing.assert_close(out.float(), _ref_packed(qkv, lens, NH), rtol=2e-2, atol=2e-2)


@pytest.mark.parametrize("B,L", [(256, 128), (1024, 128), (1024, 256)])
def test_large_msra_batches(B, L):
    """MSRA-shaped batches of thousands of tiles; each sequence's context is also byte-identical to the one it gets when
    it is the whole batch."""
    NH = 12
    lens = [int(n) for n in synthetic.msra_lengths(B, L, np.random.default_rng(B + L))]
    lens[B // 2] = L                                           # one sequence at the bound, wherever MSRA lengths stop
    qkv = _qkv(sum(lens), NH, seed=B + L)
    out = _attend(qkv, NH, lens)
    assert torch.isfinite(out.float()).all()
    torch.testing.assert_close(out.float(), _ref_packed(qkv, lens, NH), rtol=2e-2, atol=2e-2)
    starts = np.concatenate([[0], np.cumsum(lens)])
    for j in (0, 1, B // 2, B - 1):
        r0, r1 = int(starts[j]), int(starts[j + 1])
        assert torch.equal(out[r0:r1], _attend(qkv[r0:r1].contiguous(), NH, [lens[j]]))


def test_no_row_of_another_sequence_leaks():
    """Every sequence of a tile-edge batch, with all other rows poisoned (huge K, NaN V), gives exactly the context it
    gets alone."""
    NH = 3
    lens = EDGE_LENS + [5, 70]
    qkv = _qkv(sum(lens), NH, seed=11)
    starts = np.concatenate([[0], np.cumsum(lens)])
    for j, n in enumerate(lens):
        r0, r1 = int(starts[j]), int(starts[j + 1])
        poisoned = qkv.clone()
        for a, b in ((0, r0), (r1, qkv.shape[0])):
            poisoned[a:b, NH * D:2 * NH * D] = 3.0e4
            poisoned[a:b, 2 * NH * D:] = float("nan")
        out = _attend(poisoned, NH, lens)
        assert torch.equal(out[r0:r1], _attend(qkv[r0:r1].contiguous(), NH, [n])), f"sequence {j} (length {n})"


@pytest.mark.parametrize("B,L", [(300, 128), (40, 200)])
def test_padded_mode_many_items(B, L):
    NH = 3
    qkv = _qkv(B * L, NH, seed=B * L)
    lens = torch.from_numpy(np.random.default_rng(B).integers(1, L + 1, B))
    mask = (torch.arange(L)[None, :] < lens[:, None]).to(torch.int32).cuda()
    ctx = _attend(qkv, NH, mask=mask, B=B, L=L)
    assert torch.isfinite(ctx.float()).all()
    q, k, v = qkv.float().view(B, L, 3, NH, D).permute(2, 0, 3, 1, 4)
    s = q @ k.transpose(-1, -2) / math.sqrt(D) + (1.0 - mask.float())[:, None, None, :] * -10000.0
    ref = (torch.softmax(s, -1) @ v).permute(0, 2, 1, 3).reshape(B * L, NH * D)
    torch.testing.assert_close(ctx.float(), ref, rtol=2e-2, atol=2e-2)
