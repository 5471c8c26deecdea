"""GPU: wgmma/TMA dense kernel vs a plain PyTorch fp32 matmul of the same bf16 operands."""
import pytest
import torch

from chinesener_b200 import ops

pytestmark = pytest.mark.gpu


def _ref(a, wt, bias, residual, epi):
    y = a.float() @ wt.float().t()
    if bias is not None:
        y = y + bias
    if epi == ops.EPI_RES_F32:
        y = y + residual
    if epi == ops.EPI_GELU_TANH_BF16:
        y = torch.nn.functional.gelu(y, approximate="tanh")
    if epi == ops.EPI_GELU_ERF_BF16:
        y = torch.nn.functional.gelu(y)
    if epi == ops.EPI_RELU_BF16:
        y = torch.relu(y)
    return y


@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (128, 256, 128), (256, 128, 768), (8192, 768, 768),
                                   (8192, 2304, 768), (1000, 768, 3072), (77, 96, 200), (4096, 3072, 768),
                                   (300, 1024, 768)])
@pytest.mark.parametrize("tile_n", [128, 192, 256, ops.TILE_2CTA_128, ops.TILE_2CTA_256])
@pytest.mark.timeout(120)
def test_gemm_matches_fp32_reference(M, N, K, tile_n):
    g = torch.Generator().manual_seed(M + N + K)
    a = torch.randn(M, K, generator=g).to(torch.bfloat16).cuda()
    wt = (torch.randn(N, K, generator=g) * 0.05).to(torch.bfloat16).cuda()
    bias = torch.randn(N, generator=g).cuda()
    out = ops.gemm_bf16(a, wt, bias, epilogue=ops.EPI_F32, tile_n=tile_n)
    ref = _ref(a, wt, bias, None, ops.EPI_F32)
    torch.testing.assert_close(out, ref, rtol=1e-4, atol=1e-3)


@pytest.mark.parametrize("tile_n", [0, ops.TILE_2CTA_256])
@pytest.mark.parametrize("epi", [ops.EPI_BF16, ops.EPI_GELU_TANH_BF16, ops.EPI_GELU_ERF_BF16, ops.EPI_RELU_BF16,
                                 ops.EPI_RES_F32])
@pytest.mark.timeout(120)
def test_gemm_epilogues(epi, tile_n):
    M, N, K = 640, 768, 512
    g = torch.Generator().manual_seed(epi)
    a = torch.randn(M, K, generator=g).to(torch.bfloat16).cuda()
    wt = (torch.randn(N, K, generator=g) * 0.05).to(torch.bfloat16).cuda()
    bias = torch.randn(N, generator=g).cuda()
    res = torch.randn(M, N, generator=g).cuda() if epi == ops.EPI_RES_F32 else None
    out = ops.gemm_bf16(a, wt, bias, residual=res, epilogue=epi, tile_n=tile_n)
    ref = _ref(a, wt, bias, res, epi)
    if out.dtype == torch.bfloat16:
        torch.testing.assert_close(out.float(), ref, rtol=1e-2, atol=1e-2)
    else:
        torch.testing.assert_close(out, ref, rtol=1e-4, atol=1e-3)


def test_gemm_rejects_misaligned_bias_and_residual():
    """The epilogue reads bias and residual as 8-byte column pairs: a view starting at an odd float is refused, not read."""
    M, N, K = 128, 128, 64
    a = torch.randn(M, K).to(torch.bfloat16).cuda()
    wt = torch.randn(N, K).to(torch.bfloat16).cuda()
    buf = torch.randn(M * N + 1).cuda()
    with pytest.raises(ops.NerB200Error):
        ops.gemm_bf16(a, wt, buf[1:N + 1], epilogue=ops.EPI_F32)
    with pytest.raises(ops.NerB200Error):
        ops.gemm_bf16(a, wt, None, residual=buf[1:].view(M, N), epilogue=ops.EPI_RES_F32)
    out = ops.gemm_bf16(a, wt, buf[2:N + 2], residual=buf[:M * N].view(M, N), epilogue=ops.EPI_RES_F32)
    torch.testing.assert_close(out, _ref(a, wt, buf[2:N + 2], buf[:M * N].view(M, N), ops.EPI_RES_F32), rtol=1e-4, atol=1e-3)


def test_gemm_auto_tile_and_no_bias():
    M, N, K = 8192, 1024, 768
    g = torch.Generator().manual_seed(1)
    a = torch.randn(M, K, generator=g).to(torch.bfloat16).cuda()
    wt = (torch.randn(N, K, generator=g) * 0.05).to(torch.bfloat16).cuda()
    out = ops.gemm_bf16(a, wt, None, epilogue=ops.EPI_F32)
    torch.testing.assert_close(out, a.float() @ wt.float().t(), rtol=1e-4, atol=1e-3)


@pytest.mark.parametrize("M,N,K", [(3150, 2304, 768), (3150, 768, 768), (3150, 3072, 768), (3150, 768, 3072), (1000, 768, 3072),
                                   (8192, 2304, 768), (128, 256, 128), (2500, 256, 3072), (3195, 1024, 64)])
@pytest.mark.parametrize("tile_n", [ops.TILE_SK_256, ops.TILE_SK_128, 0])
@pytest.mark.timeout(120)
def test_gemm_stream_k_matches_fp32_reference(M, N, K, tile_n):
    """Stream-K scheduling (split tiles summed through the fp32 scratch): same result as whole-tile
    scheduling, call after call (the finisher restores the flags), fp32 and bf16 outputs."""
    g = torch.Generator().manual_seed(M + N + K)
    a = torch.randn(M, K, generator=g).to(torch.bfloat16).cuda()
    wt = (torch.randn(N, K, generator=g) * 0.05).to(torch.bfloat16).cuda()
    bias = torch.randn(N, generator=g).cuda()
    res = torch.randn(M, N, generator=g).cuda()
    ref = _ref(a, wt, bias, None, ops.EPI_F32)
    for _ in range(3):
        out = ops.gemm_bf16(a, wt, bias, epilogue=ops.EPI_F32, tile_n=tile_n)
        torch.testing.assert_close(out, ref, rtol=1e-4, atol=1e-3)
    out = ops.gemm_bf16(a, wt, bias, residual=res, epilogue=ops.EPI_RES_F32, tile_n=tile_n)
    torch.testing.assert_close(out, ref + res, rtol=1e-4, atol=1e-3)
    out = ops.gemm_bf16(a, wt, bias, epilogue=ops.EPI_GELU_TANH_BF16, tile_n=tile_n)
    torch.testing.assert_close(out.float(), _ref(a, wt, bias, None, ops.EPI_GELU_TANH_BF16), rtol=1e-2, atol=1e-2)


def test_gemm_stream_k_on_a_second_stream():
    M, N, K = 3150, 768, 3072
    g = torch.Generator().manual_seed(5)
    a = torch.randn(M, K, generator=g).to(torch.bfloat16).cuda()
    wt = (torch.randn(N, K, generator=g) * 0.05).to(torch.bfloat16).cuda()
    ref = a.float() @ wt.float().t()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        o2 = ops.gemm_bf16(a, wt, None, epilogue=ops.EPI_F32, tile_n=ops.TILE_SK_256)
    o1 = ops.gemm_bf16(a, wt, None, epilogue=ops.EPI_F32, tile_n=ops.TILE_SK_256)
    torch.cuda.synchronize()
    torch.testing.assert_close(o1, ref, rtol=1e-4, atol=1e-3)
    torch.testing.assert_close(o2, ref, rtol=1e-4, atol=1e-3)


@pytest.mark.parametrize("rows", [3150, 64, 1, 200, 4097])
def test_grouped_mn_major_weight_gradients(rows):
    """ner_wgrad_group_bf16: dW += X^T dY for a group of problems in one launch, operands consumed token-major (MN-major
    wgmma descriptors, no transposed copies) — vs fp32 matmuls of the same bf16 operands; accumulation into dW, column
    slices of a fused dY (the Q/K/V gradients), rows that are not a multiple of the 64-token k-block."""
    g = torch.Generator().manual_seed(rows)
    H, I = 768, 3072
    x16 = torch.randn(rows, H, generator=g).to(torch.bfloat16).cuda()
    ctx = torch.randn(rows, H, generator=g).to(torch.bfloat16).cuda()
    inter = torch.randn(rows, I, generator=g).to(torch.bfloat16).cuda()
    dqkv = (torch.randn(rows, 3 * H, generator=g) * 0.1).to(torch.bfloat16).cuda()
    dz = (torch.randn(rows, H, generator=g) * 0.1).to(torch.bfloat16).cuda()
    dpre = (torch.randn(rows, I, generator=g) * 0.1).to(torch.bfloat16).cuda()
    dws = [torch.randn(a, b, generator=g).cuda() for a, b in ((H, H), (H, H), (H, H), (H, H), (H, I), (I, H))]
    want = [w.clone() for w in dws]
    probs = [(x16, dqkv, 0, dws[0]), (x16, dqkv, H, dws[1]), (x16, dqkv, 2 * H, dws[2]), (ctx, dz, 0, dws[3]),
             (x16, dpre, 0, dws[4]), (inter, dz, 0, dws[5])]
    ops.wgrad_group(probs, rows)
    for (x, dy, c0, _), w0, got in zip(probs, want, dws):
        ref = w0 + x.float().t() @ dy[:, c0:c0 + w0.shape[1]].float()
        scale = ref.abs().max().item()
        err = (got - ref).abs().max().item()
        assert err < 2e-4 * max(1.0, scale), (rows, tuple(w0.shape), c0, err, scale)
