"""GPU: every epilogue mode of ner_gemm_bf16 under every tile it accepts, at row counts and widths where the TMA store of
the output chunks is clipped — a row tail inside a 64-row warpgroup slice (M = 1, 127, 129, 3549), a 64-column bf16 chunk
only half inside the matrix (N = 96) and partial last N tiles (N = 768 / 2304 under 256- and 192-wide tiles)."""
import pytest
import torch

from chinesener_b200 import ops
from chinesener_b200._lib import check, lib, ptr, stream

pytestmark = pytest.mark.gpu

TILES = [64, 128, 192, 256, ops.TILE_2CTA_128, ops.TILE_2CTA_256, ops.TILE_SK_128, ops.TILE_SK_256, 0,
         ops.TILE_AUTO_THROUGHPUT]
EPIS = [ops.EPI_F32, ops.EPI_BF16, ops.EPI_GELU_TANH_BF16, ops.EPI_GELU_ERF_BF16, ops.EPI_RELU_BF16, ops.EPI_RES_F32,
        ops.EPI_RES_RELU_F32, ops.EPI_DIAG_DISCARD]
F32_OUT = (ops.EPI_F32, ops.EPI_RES_F32, ops.EPI_RES_RELU_F32)
K = 192

_operands = {}


def _inputs(M, N):
    if (M, N) not in _operands:
        g = torch.Generator(device="cuda").manual_seed(M * 7919 + N)
        a = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
        wt = (torch.randn(N, K, device="cuda", generator=g) * 0.1).to(torch.bfloat16)
        bias = torch.randn(N, device="cuda", generator=g)
        res = torch.randn(M, N, device="cuda", generator=g)
        y = a.float() @ wt.float().t() + bias
        _operands.clear()
        _operands[(M, N)] = (a, wt, bias, res, y)
    return _operands[(M, N)]


def _ref(y, res, epi):
    if epi in (ops.EPI_RES_F32, ops.EPI_RES_RELU_F32):
        y = y + res
    if epi == ops.EPI_GELU_TANH_BF16:
        y = torch.nn.functional.gelu(y, approximate="tanh")
    elif epi == ops.EPI_GELU_ERF_BF16:
        y = torch.nn.functional.gelu(y)
    elif epi in (ops.EPI_RELU_BF16, ops.EPI_RES_RELU_F32):
        y = torch.relu(y)
    return y


@pytest.mark.parametrize("N", [96, 768, 2304])
@pytest.mark.parametrize("M", [1, 127, 129, 3549])
@pytest.mark.parametrize("epi", EPIS)
@pytest.mark.parametrize("tile_n", TILES)
@pytest.mark.timeout(120)
def test_gemm_epilogue_store_clipping(tile_n, epi, M, N):
    a, wt, bias, res, y = _inputs(M, N)
    odt = torch.float32 if epi in F32_OUT else torch.bfloat16
    # one guard row before and after the output: a store that is not clipped to [M, N] lands there
    buf = torch.full((M + 2, N), 7.0, device="cuda", dtype=odt)
    out = buf[1:M + 1]
    # the C entry point directly, so that the guarded view is the output of every mode, the diagnostic one included
    check(lib().ner_gemm_bf16(ptr(a), ptr(wt), ptr(bias), ptr(res), ptr(out), M, N, K, epi, tile_n, stream()))
    torch.cuda.synchronize()
    assert bool((buf[0] == 7.0).all()) and bool((buf[M + 1] == 7.0).all()), "store outside the output rows"
    if epi == ops.EPI_DIAG_DISCARD:
        assert bool((out == 7.0).all()), "the diagnostic mode stores nothing"
        return
    ref = _ref(y, res, epi)
    if odt == torch.bfloat16:
        torch.testing.assert_close(out.float(), ref, rtol=1e-2, atol=1e-2)
    else:
        torch.testing.assert_close(out, ref, rtol=1e-4, atol=1e-3)
