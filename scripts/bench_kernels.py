"""Stand-alone kernel timings (CUDA events) used while tuning; not the driver's bench.py.

usage: python scripts/bench_kernels.py [crf] [gemm] [attn] [wgrad] [--lib OTHER/libner_b200.so]
"""
import json
import os
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
    from chinesener_b200 import _lib
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    out["viterbi_plan"] = _lib.VIT_PLANS[_lib.lib().ner_crf_viterbi_plan(B, L, K, x.data_ptr() % 16 == 0, sms)]
    for exact in (False, True):
        med, best = timeit(lambda: ops.crf_loglik_fwd(x, tags, lens, tr, exact=exact))
        byts = B * L * (4 * K + 4) + 8 * B + 4 * K * K
        out["loglik_fwd_exact" if exact else "loglik_fwd"] = dict(ms=med, best_ms=best, GBps=byts / med / 1e6, bytes=byts)
    # latency regime
    xs, ls, ts = x[:64].contiguous(), lens[:64].contiguous(), tags[:64].contiguous()
    out["viterbi_B64_us"] = timeit(lambda: ops.crf_viterbi(xs, ls, tr), iters=50)[0] * 1e3
    out["loglik_B64_us"] = timeit(lambda: ops.crf_loglik_fwd(xs, ts, ls, tr), iters=50)[0] * 1e3
    return out


BF16_PEAK_TFLOPS = 989.0     # H100 SXM data sheet, dense bf16, 700 W
# the GEMMs of one bert_bilstm_crf PREDICT step: (name, N, K, epilogue, launches per step)
STEP_GEMMS = [("qkv", 2304, 768, ops.EPI_BF16, 12), ("out", 768, 768, ops.EPI_BF16, 12),
              ("ffn1", 3072, 768, ops.EPI_GELU_TANH_BF16, 12), ("ffn2", 768, 3072, ops.EPI_BF16, 12),
              ("lstm_x", 1024, 768, ops.EPI_F32, 1)]
# packed tokens of bench.py's first batch (seed 1234) and of its four batches stacked
STEP_ROWS = (3549, 12202)
EPI_NAMES = {ops.EPI_BF16: "bf16", ops.EPI_GELU_TANH_BF16: "gelu_tanh", ops.EPI_F32: "f32", ops.EPI_DIAG_DISCARD: "discard"}


def device_card():
    """Card name, power limit and max SM clock, read in the same process as the timings."""
    import subprocess
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    except (OSError, subprocess.SubprocessError):
        q = []
    return {"torch_name": torch.cuda.get_device_name(), "nvidia_smi": q[0] if q else None}


def _gemm_fn(lib_path):
    """ner_gemm_bf16 of the package's library, or of another build of it (`--lib`) for an A/B in one process.  Called
    through ctypes directly, so that DISCARD can run on the output buffer of the epilogue it is compared with."""
    import ctypes
    from chinesener_b200 import _lib
    if lib_path is None:
        fn = _lib.lib().ner_gemm_bf16
    else:
        fn = ctypes.CDLL(os.path.abspath(lib_path)).ner_gemm_bf16
        fn.restype, fn.argtypes = _lib.SIGNATURES["ner_gemm_bf16"]

    def call(a, w, bias, o, epi, tn):
        M, K = a.shape
        rc = fn(a.data_ptr(), w.data_ptr(), bias.data_ptr(), None, o.data_ptr(), M, w.shape[0], K, epi, tn, _lib.stream())
        if rc != 0:
            raise RuntimeError(f"{lib_path}: ner_gemm_bf16 returned {rc}")
        return o
    return call


def bench_gemm(lib_path=None, iters=20):
    """The step's GEMM shapes at one batch / four stacked batches of packed tokens, each with its own epilogue and with
    NER_EPI_DIAG_DISCARD (accumulate, store nothing), under tile_n = 0 and TILE_AUTO_THROUGHPUT.  `exposure_us` =
    t(epilogue) - t(discard): the time the epilogue adds to the mainloop.  With `lib_path` the same launches of that
    library are timed alternately with this one ("ref") and the outputs compared byte for byte."""
    libs = {"new": _gemm_fn(None)}
    if lib_path:
        libs["ref"] = _gemm_fn(lib_path)
    out = {"card": device_card(), "peak_tflops": BF16_PEAK_TFLOPS, "rows": {}, "per_batch_us": {}}
    g = torch.Generator(device="cuda").manual_seed(1234)
    for M in STEP_ROWS:
        for tn in (0, ops.TILE_AUTO_THROUGHPUT):
            for name, N, K, epi, reps in STEP_GEMMS:
                a = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
                w = (torch.randn(N, K, device="cuda", generator=g) * 0.05).to(torch.bfloat16)
                bias = torch.randn(N, device="cuda", generator=g)
                odt = torch.float32 if epi == ops.EPI_F32 else torch.bfloat16
                flops = 2.0 * M * N * K
                row = {"M": M, "N": N, "K": K, "tile_n": tn, "epilogue": EPI_NAMES[epi]}
                outs = {}
                for tag, fn in libs.items():
                    o = torch.empty(M, N, device="cuda", dtype=odt)
                    fn(a, w, bias, o, epi, tn)
                    outs[tag] = o.clone()
                # alternate the libraries launch set by launch set, so drift in clocks hits both alike
                for tag, fn in libs.items():
                    for e in (epi, ops.EPI_DIAG_DISCARD):
                        o = torch.empty(M, N, device="cuda", dtype=odt)
                        med, _ = timeit(lambda: fn(a, w, bias, o, e, tn), iters=iters)
                        row[f"{tag}_{EPI_NAMES[e]}_us"] = round(med * 1e3, 2)
                    t_ep, t_d = row[f"{tag}_{EPI_NAMES[epi]}_us"], row[f"{tag}_discard_us"]
                    row[f"{tag}_TFLOPs"] = round(flops / t_ep / 1e6, 1)
                    row[f"{tag}_frac_peak"] = round(flops / t_ep / 1e6 / BF16_PEAK_TFLOPS, 3)
                    row[f"{tag}_discard_frac_peak"] = round(flops / t_d / 1e6 / BF16_PEAK_TFLOPS, 3)
                    row[f"{tag}_exposure_us"] = round(t_ep - t_d, 2)
                    row[f"{tag}_exposure_share"] = round((t_ep - t_d) / t_ep, 3)
                    key = f"M{M}_t{tn}_{tag}"
                    out["per_batch_us"][key] = round(out["per_batch_us"].get(key, 0.0) + reps * t_ep, 1)
                if "ref" in outs:
                    row["bytes_equal_ref"] = bool(torch.equal(outs["new"].view(torch.uint8), outs["ref"].view(torch.uint8)))
                    row["max_abs_diff_ref"] = float((outs["new"].float() - outs["ref"].float()).abs().max())
                out["rows"][f"{name}_M{M}_t{tn}"] = row
    # every explicit tile of this library at the same shapes: what the tile_n = 0 cost model chooses between
    out["tiles_us"] = {}
    for M in STEP_ROWS:
        for name, N, K, epi, _ in STEP_GEMMS:
            a = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
            w = (torch.randn(N, K, device="cuda", generator=g) * 0.05).to(torch.bfloat16)
            bias = torch.randn(N, device="cuda", generator=g)
            o = torch.empty(M, N, device="cuda", dtype=torch.float32 if epi == ops.EPI_F32 else torch.bfloat16)
            times = {}
            for tn in (0, 128, 192, 256, ops.TILE_SK_128, ops.TILE_SK_256, ops.TILE_2CTA_256):
                if tn in (192,) and N % 192:
                    continue
                times[str(tn)] = round(timeit(lambda: libs["new"](a, w, bias, o, epi, tn), iters=iters)[0] * 1e3, 2)
            out["tiles_us"][f"{name}_M{M}"] = times
    return out


def _attention_fn(lib_path):
    """ner_bert_attention (packed mode, inference) of the package's library, or of another build of it (`--lib`)."""
    import ctypes
    from chinesener_b200 import _lib
    if lib_path is None:
        fn = _lib.lib().ner_bert_attention
    else:
        fn = ctypes.CDLL(os.path.abspath(lib_path)).ner_bert_attention
        fn.restype, fn.argtypes = _lib.SIGNATURES["ner_bert_attention"]

    def call(qkv, cu, ctx, B, L, NH):
        rc = fn(qkv.data_ptr(), None, ctx.data_ptr(), B, L, NH, 64, 0.125, -10000.0, cu.data_ptr(), qkv.shape[0], 1.0, 0,
                _lib.stream())
        if rc != 0:
            raise RuntimeError(f"{lib_path}: ner_bert_attention returned {rc}")
        return ctx
    return call


def bench_attention(lib_path=None, rounds=3):
    """wgmma attention vs the mma.sync kernel at the bench shapes: one MSRA-shaped 64-sentence batch and four stacked.
    With `lib_path` the same call of that library ("ref") is timed alternately with this one, round by round, and the
    contexts (written over NaN) are compared byte for byte."""
    from chinesener_b200 import synthetic
    import numpy as np
    libs = {"new": _attention_fn(None)}
    if lib_path:
        libs["ref"] = _attention_fn(lib_path)
    out = {"card": device_card()}
    NH, D = 12, 64
    for B in (64, 256):
        lens = synthetic.msra_lengths(B, 128, np.random.default_rng(1234))
        T = int(lens.sum())
        qkv = torch.randn(T, 3 * NH * D, device="cuda").to(torch.bfloat16)
        cu = torch.tensor([0] + list(np.cumsum(lens)), dtype=torch.int32, device="cuda")
        ctx = torch.full((T, NH * D), float("nan"), device="cuda", dtype=torch.bfloat16)
        flops = 4.0 * float((lens.astype(np.float64) ** 2).sum()) * NH * D
        row = {"tokens": T}
        outs = {}
        for tag, fn in libs.items():
            outs[tag] = fn(qkv, cu, ctx.clone(), B, 128, NH)
        row["finite"] = bool(torch.isfinite(outs["new"].float()).all())
        if "ref" in outs:
            row["bytes_equal_ref"] = bool(torch.equal(outs["new"].view(torch.uint8), outs["ref"].view(torch.uint8)))
            row["max_abs_diff_ref"] = float((outs["new"].float() - outs["ref"].float()).abs().max())
        runs = [(tag, fn, None) for tag, fn in libs.items()] + [("mma_sync", libs["new"], "1")]
        meds = {name: [] for name, _, _ in runs}
        for _ in range(rounds):
            for name, fn, var in runs:
                if var:
                    os.environ["NER_ATTN_VARIANT"] = var
                try:
                    meds[name].append(timeit(lambda: fn(qkv, cu, ctx, B, 128, NH), iters=30)[0] * 1e3)
                finally:
                    os.environ.pop("NER_ATTN_VARIANT", None)
        for name, ts in meds.items():
            us = min(ts)
            row[name] = dict(us=round(us, 2), round_us=[round(t, 2) for t in ts], TFLOPs=round(flops / us / 1e6, 1))
        if "ref" in meds:
            row["speedup_vs_ref"] = round(row["ref"]["us"] / row["new"]["us"], 2)
        out[f"B{B}"] = row
    return out


def print_gemm_table(res):
    print(f"# card: {res['card']}")
    tags = [t for t in ("new", "ref") if any(f"{t}_TFLOPs" in r for r in res["rows"].values())]
    hdr = f"{'gemm':24s} {'epi':9s}" + "".join(f" | {t:>3s}: {'us':>8s} {'disc us':>8s} {'TF/s':>6s} {'frac':>5s} {'d.frac':>6s} "
                                              f"{'expo us':>8s} {'share':>5s}" for t in tags)
    print(hdr)
    for k, r in res["rows"].items():
        line = f"{k:24s} {r['epilogue']:9s}"
        for t in tags:
            t_ep = r[f"{t}_{r['epilogue']}_us"]
            line += (f" | {t:>3s}: {t_ep:8.1f} "
                     f"{r[f'{t}_discard_us']:8.1f} {r[f'{t}_TFLOPs']:6.1f} {r[f'{t}_frac_peak']:5.2f} "
                     f"{r[f'{t}_discard_frac_peak']:6.2f} {r[f'{t}_exposure_us']:8.1f} {r[f'{t}_exposure_share']:5.2f}")
        if "bytes_equal_ref" in r:
            line += f" | bytes_equal={r['bytes_equal_ref']} maxdiff={r['max_abs_diff_ref']:.3g}"
        print(line)
    print("# GEMM kernel us per step (12 layers x 4 + lstm_x, sum of isolated launches):", res["per_batch_us"])
    print("# us per explicit tile_n (this library, step epilogue):")
    for k, v in res["tiles_us"].items():
        print(f"{k:16s} " + " ".join(f"{t}={us}" for t, us in v.items()))


if __name__ == "__main__":
    argv = sys.argv[1:]
    lib_path = None
    if "--lib" in argv:                 # --lib PATH: time / compare gemm / attn of another libner_b200.so as well
        i = argv.index("--lib")
        lib_path = argv[i + 1]
        del argv[i:i + 2]
    which = argv or ["crf", "gemm"]
    res = {}
    if "crf" in which:
        res["crf"] = bench_crf()
    if "gemm" in which:
        res["gemm"] = bench_gemm(lib_path)
        print_gemm_table(res["gemm"])
    if "attn" in which:
        res["attention"] = bench_attention(lib_path)
    print(json.dumps(res, indent=1))


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
