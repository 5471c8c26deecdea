"""Stand-alone kernel timings (CUDA events) used while tuning; not the driver's bench.py.

usage: python scripts/bench_kernels.py [crf] [gemm]
"""
import json
import sys

import torch

sys.path.insert(0, __import__("os").path.dirname(__import__("os").path.dirname(__import__("os").path.abspath(__file__))))
from chinesener_b200 import ops  # noqa: E402


def timeit(fn, warm=3, iters=10):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    # park the GPU behind a ~4 ms spin kernel so the host enqueues every timed launch before the first one
    # starts: the event pairs then bracket kernel execution, not the Python/driver launch latency (~18 us/call)
    torch.cuda._sleep(8_000_000)
    for s, e in evs:
        s.record()
        fn()
        e.record()
    torch.cuda.synchronize()
    ts = sorted(s.elapsed_time(e) for s, e in evs)
    return ts[len(ts) // 2], ts[0]


def bench_crf(B=262144, L=128, K=10):
    g = torch.Generator(device="cuda").manual_seed(1234)
    x = torch.randn(B, L, K, device="cuda", generator=g)
    tr = torch.randn(K, K, device="cuda", generator=g) * 0.5
    lens = torch.full((B,), L, dtype=torch.int32, device="cuda")
    tags = torch.randint(0, K, (B, L), device="cuda", dtype=torch.int32)
    out = {}
    med, best = timeit(lambda: ops.crf_viterbi(x, lens, tr))
    byts = B * L * (4 * K) + 4 * B + 4 * K * K + B * L * 4 + 4 * B
    out["viterbi"] = dict(ms=med, best_ms=best, GBps=byts / med / 1e6, bytes=byts)
    import os
    out["fwd_variant"] = os.environ.get("NER_CRF_FWD_VARIANT", "0")
    out["vit_variant"] = os.environ.get("NER_CRF_VIT_VARIANT", "0")
    for exact in (False, True):
        med, best = timeit(lambda: ops.crf_loglik_fwd(x, tags, lens, tr, exact=exact))
        byts = B * L * (4 * K + 4) + 8 * B + 4 * K * K
        out["loglik_fwd_exact" if exact else "loglik_fwd"] = dict(ms=med, best_ms=best, GBps=byts / med / 1e6, bytes=byts)
    # latency regime
    xs, ls, ts = x[:64].contiguous(), lens[:64].contiguous(), tags[:64].contiguous()
    out["viterbi_B64_us"] = timeit(lambda: ops.crf_viterbi(xs, ls, tr), iters=50)[0] * 1e3
    out["loglik_B64_us"] = timeit(lambda: ops.crf_loglik_fwd(xs, ts, ls, tr), iters=50)[0] * 1e3
    return out


def bench_gemm(packed_only=False, iters=20):
    out = {}
    shapes = [(8192, 2304, 768), (8192, 768, 768), (8192, 3072, 768), (8192, 768, 3072), (3150, 2304, 768),
              (3150, 768, 768), (3150, 3072, 768), (3150, 768, 3072), (3150, 1024, 768)]
    if packed_only:
        shapes = [s for s in shapes if s[0] == 3150 and s[1] != 1024]
    for (M, N, K) in shapes:
        a = torch.randn(M, K, device="cuda").to(torch.bfloat16)
        w = (torch.randn(N, K, device="cuda") * 0.05).to(torch.bfloat16)
        bias = torch.randn(N, device="cuda")
        res = torch.randn(M, N, device="cuda")
        for tn in (0, 128, 192, 256, ops.TILE_2CTA_256, ops.TILE_SK_256, ops.TILE_SK_128):
            for epi, nm in ((ops.EPI_BF16, "bf16"), (ops.EPI_F32, "f32")):
                o = torch.empty(M, N, device="cuda", dtype=torch.float32 if epi in (ops.EPI_RES_F32, ops.EPI_F32) else torch.bfloat16)
                med, best = timeit(lambda: ops.gemm_bf16(a, w, bias, residual=res if epi == ops.EPI_RES_F32 else None,
                                                         epilogue=epi, tile_n=tn, out=o), iters=iters)
                out[f"{M}x{N}x{K}_t{tn}_{nm}"] = dict(us=round(med * 1e3, 1), TFLOPs=round(2.0 * M * N * K / med / 1e9, 1))
    return out


if __name__ == "__main__":
    which = sys.argv[1:] or ["crf", "gemm"]
    res = {}
    if "crf" in which:
        res["crf"] = bench_crf()
    if "gemm" in which:
        res["gemm"] = bench_gemm()
    if "gemm_packed" in which:          # short run for an ncu launch list (true per-kernel durations)
        res["gemm"] = bench_gemm(packed_only=True, iters=3)
    print(json.dumps(res, indent=1))


def bench_attention():
    """wgmma attention vs the mma.sync kernel at the bench shapes: one MSRA-shaped 64-sentence batch and four stacked."""
    import os
    from chinesener_b200 import synthetic
    import numpy as np
    out = {}
    NH, D = 12, 64
    for B in (64, 256):
        lens = synthetic.msra_lengths(B, 128, np.random.default_rng(1234))
        T = int(lens.sum())
        qkv = torch.randn(T, 3 * NH * D, device="cuda").to(torch.bfloat16)
        cu = torch.tensor([0] + list(np.cumsum(lens)), dtype=torch.int32, device="cuda")
        for name, var in (("wgmma", None), ("mma_sync", "1")):
            if var:
                os.environ["NER_ATTN_VARIANT"] = var
            med, best = timeit(lambda: ops.bert_attention(qkv, None, B, 128, NH, D, cu_seqlens=cu), iters=30)
            os.environ.pop("NER_ATTN_VARIANT", None)
            flops = 4.0 * float((lens.astype(np.float64) ** 2).sum()) * NH * D
            out[f"{name}_B{B}"] = dict(us=round(med * 1e3, 2), best_us=round(best * 1e3, 2), tokens=T, TFLOPs=round(flops / med / 1e9, 1))
    return out


if __name__ == "__main__" and "attn" in sys.argv[1:]:
    print(json.dumps({"attention": bench_attention()}, indent=1))


def bench_wgrad(rows=3150):
    """One encoder layer's weight gradients: grouped MN-major launch vs the transposes + four GEMMs it replaces."""
    H, I = 768, 3072
    x16, ctx = (torch.randn(rows, H, device="cuda").to(torch.bfloat16) for _ in range(2))
    inter = torch.randn(rows, I, device="cuda").to(torch.bfloat16)
    dqkv = torch.randn(rows, 3 * H, device="cuda").to(torch.bfloat16)
    dz = torch.randn(rows, H, device="cuda").to(torch.bfloat16)
    dpre = torch.randn(rows, I, device="cuda").to(torch.bfloat16)
    dws = [torch.zeros(a, b, device="cuda") for a, b in ((H, H), (H, H), (H, H), (H, H), (H, I), (I, H))]
    probs = [(x16, dqkv, 0, dws[0]), (x16, dqkv, H, dws[1]), (x16, dqkv, 2 * H, dws[2]), (ctx, dz, 0, dws[3]),
             (x16, dpre, 0, dws[4]), (inter, dz, 0, dws[5])]
    flops = 2.0 * rows * (3 * H * H + H * H + 2 * H * I)
    med, best = timeit(lambda: ops.wgrad_group(probs, rows), iters=20)
    out = {"grouped_mn_major": dict(us=round(med * 1e3, 1), TFLOPs=round(flops / med / 1e9, 1))}
    dw_qkv = torch.zeros(H, 3 * H, device="cuda")

    def old():
        ops.wgrad_gemm_bf16(x16, dqkv, dw_qkv)
        ops.wgrad_gemm_bf16(ctx, dz, dws[3])
        ops.wgrad_gemm_bf16(x16, dpre, dws[4])
        ops.wgrad_gemm_bf16(inter, dz, dws[5])
    med, best = timeit(old, iters=20)
    out["transposes_plus_4_gemms"] = dict(us=round(med * 1e3, 1), TFLOPs=round(flops / med / 1e9, 1))
    return out


if __name__ == "__main__" and "wgrad" in sys.argv[1:]:
    print(json.dumps({"wgrad": bench_wgrad()}, indent=1))
