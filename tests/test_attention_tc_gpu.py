"""GPU: the wgmma attention kernel (csrc/attention_tc.cu — S = Q K^T and O = P V in registers, TMA operand loads, V as
an MN-major operand) against a plain PyTorch fp32 softmax(QK^T)V of the same bf16 inputs, against the warp-level mma.sync
kernel it replaces on the inference path, on ragged packed batches, and with hostile neighbours (rows of other sequences
that ride along in a TMA box must never leak into a result)."""
import math
import os

import pytest
import torch

from chinesener_b200 import ops

pytestmark = pytest.mark.gpu
D = 64


def _ref_packed(qkv, lens, NH):
    out, r0 = [], 0
    for n in lens:
        q, k, v = qkv[r0:r0 + n].float().view(n, 3, NH, D).permute(1, 2, 0, 3)
        s = q @ k.transpose(-1, -2) / math.sqrt(D)
        out.append((torch.softmax(s, -1) @ v).permute(1, 0, 2).reshape(n, NH * D))
        r0 += n
    return torch.cat(out)


@pytest.mark.parametrize("lens,NH", [([128, 1, 31, 32, 33, 64, 65, 127], 12), ([129, 200, 256, 2, 255], 3), ([5], 1),
                                     ([150] * 4 + [17], 12), ([64] * 9, 2)])
def test_packed_ragged_lengths(lens, NH):
    g = torch.Generator().manual_seed(sum(lens) + NH)
    T = sum(lens)
    qkv = torch.randn(T, 3 * NH * D, generator=g).to(torch.bfloat16).cuda()
    cu = torch.tensor([0] + list(torch.tensor(lens).cumsum(0)), dtype=torch.int32).cuda()
    out = ops.bert_attention(qkv, None, len(lens), max(lens), NH, D, cu_seqlens=cu)
    ref = _ref_packed(qkv, lens, NH)
    torch.testing.assert_close(out.float(), ref, rtol=2e-2, atol=2e-2)
    os.environ["NER_ATTN_VARIANT"] = "1"                      # the mma.sync kernel on the same inputs
    try:
        old = ops.bert_attention(qkv, None, len(lens), max(lens), NH, D, cu_seqlens=cu)
    finally:
        del os.environ["NER_ATTN_VARIANT"]
    torch.testing.assert_close(out.float(), old.float(), rtol=2e-2, atol=2e-2)


def test_rows_of_other_sequences_never_leak():
    """Sequence 0 is short; the rows that follow it inside its 64-row TMA boxes belong to sequence 1, whose K is huge and
    whose V is +inf / NaN.  Sequence 0's context must be exactly what it is when it stands alone."""
    NH = 2
    g = torch.Generator().manual_seed(3)
    lens = [19, 90]
    qkv = torch.randn(sum(lens), 3 * NH * D, generator=g).to(torch.bfloat16)
    alone = ops.bert_attention(qkv[:19].contiguous().cuda(), None, 1, 19, NH, D,
                               cu_seqlens=torch.tensor([0, 19], dtype=torch.int32).cuda())
    poisoned = qkv.clone()
    poisoned[19:, NH * D:2 * NH * D] = 3.0e4                   # K of the neighbour: huge scores if they leaked
    poisoned[19:60, 2 * NH * D:] = float("inf")                # V of the neighbour
    poisoned[60:, 2 * NH * D:] = float("nan")
    cu = torch.tensor([0, 19, 109], dtype=torch.int32).cuda()
    out = ops.bert_attention(poisoned.cuda(), None, 2, 90, NH, D, cu_seqlens=cu)
    assert torch.equal(out[:19], alone)
    assert torch.isfinite(out[:19].float()).all()


@pytest.mark.parametrize("B,L", [(3, 128), (2, 96), (2, 200)])
def test_padded_mode_uses_the_additive_mask(B, L):
    NH = 4
    g = torch.Generator().manual_seed(B * L)
    qkv = torch.randn(B * L, 3 * NH * D, generator=g).to(torch.bfloat16).cuda()
    lens = torch.tensor([L] + [max(1, L // (i + 2)) for i in range(B - 1)])
    mask = (torch.arange(L)[None, :] < lens[:, None]).to(torch.int32).cuda()
    ctx = ops.bert_attention(qkv, mask, B, L, NH, D)
    q, k, v = qkv.float().view(B, L, 3, NH, D).permute(2, 0, 3, 1, 4)
    s = q @ k.transpose(-1, -2) / math.sqrt(D) + (1.0 - mask.float())[:, None, None, :] * -10000.0
    ref = (torch.softmax(s, -1) @ v).permute(0, 2, 1, 3).reshape(B * L, NH * D)
    torch.testing.assert_close(ctx.float(), ref, rtol=2e-2, atol=2e-2)


def test_peaked_and_flat_rows():
    """softmax extremes: one dominant key (p -> 1 for it, exact 0 mass elsewhere after bf16) and all-equal scores."""
    NH, L = 1, 128
    qkv = torch.zeros(L, 3 * D, dtype=torch.float32)
    qkv[:, 2 * D:] = torch.arange(L, dtype=torch.float32)[:, None] / 8.0        # V row k = k/8
    qkv[0, :D] = 30.0                                                       # query 0 looks for key 7
    qkv[7, D:2 * D] = 30.0
    out = ops.bert_attention(qkv.to(torch.bfloat16).cuda(), None, 1, L, NH, D,
                             cu_seqlens=torch.tensor([0, L], dtype=torch.int32).cuda()).float().cpu()
    assert torch.allclose(out[0], torch.full((D,), 7 / 8.0), atol=1e-2)
    assert torch.allclose(out[1:], torch.full((L - 1, D), (L - 1) / 16.0), rtol=1e-2)    # uniform attention: mean of V
