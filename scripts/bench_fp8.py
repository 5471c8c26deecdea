"""bf16 vs FP8 (bert_precision='fp8') on the encoder: GEMMs, LayerNorm, the 12-layer encoder and two plugins' PREDICT, in
one process, with the card, power limit and SM clock read in the same run.

    python scripts/bench_fp8.py [--reps 5] [--iters 50]

Rates are shares of the H100 SXM data-sheet dense peaks (989 TFLOP/s bf16, 1979 TFLOP/s fp8, both for a 700 W card).
Each pair of variants is timed alternately, `--reps` times, and the median is reported.
"""
import argparse
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from chinesener_b200 import bert, engine, ops, synthetic, variables  # noqa: E402
from chinesener_b200.tools import layer  # noqa: E402

PEAK = {"bf16": 989e12, "fp8": 1979e12}
GEMMS = [("qkv", 2304, 768), ("ffn1", 3072, 768), ("ffn2", 768, 3072)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def timed(fn, iters):
    """ms per call: CUDA events around `iters` back-to-back calls after a warm-up call."""
    fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def alternate(fns, reps, iters):
    """{name: median ms} timing the variants in turn, `reps` rounds."""
    t = {k: [] for k in fns}
    for _ in range(reps):
        for k, f in fns.items():
            t[k].append(timed(f, iters))
    return {k: sorted(v)[len(v) // 2] for k, v in t.items()}


def bench_gemms(reps, iters):
    print("\n| GEMM | rows | bf16 µs | bf16 TFLOP/s | share of 989 | fp8 µs | fp8 TFLOP/s | share of 1979 | fp8 speed-up |")
    print("|---|---|---|---|---|---|---|---|---|")
    g = torch.Generator(device="cuda").manual_seed(0)
    for rows in (3549, 12202):
        for name, N, K in GEMMS:
            a = torch.randn(rows, K, device="cuda", generator=g)
            w = torch.randn(K, N, device="cuda", generator=g) * 0.03
            bias = torch.zeros(N, device="cuda")
            a16, w16 = a.to(torch.bfloat16), ops.pack_weight_bf16(w)
            import _fp8_oracle as fo
            qa, sa = (t.cuda() for t in fo.quantize_rows(a))
            qw, sw = ops.quantize_weight_e4m3(w)
            gelu = name == "ffn1"
            e16 = ops.EPI_GELU_TANH_BF16 if gelu else ops.EPI_BF16
            e8 = ops.EPI_GELU_TANH_E4M3 if gelu else ops.EPI_BF16
            t = alternate({"bf16": lambda: ops.gemm_bf16(a16, w16, bias, epilogue=e16),
                           "fp8": lambda: ops.gemm_e4m3(qa, sa, qw, sw, bias, epilogue=e8)}, reps, iters)
            fl = 2.0 * rows * N * K
            r16, r8 = fl / (t["bf16"] * 1e-3), fl / (t["fp8"] * 1e-3)
            print(f"| {name} {N}x{K} | {rows} | {1e3 * t['bf16']:.1f} | {r16 / 1e12:.0f} | {r16 / PEAK['bf16']:.2f} | "
                  f"{1e3 * t['fp8']:.1f} | {r8 / 1e12:.0f} | {r8 / PEAK['fp8']:.2f} | {t['bf16'] / t['fp8']:.2f}x |")


def bench_layernorm(reps, iters):
    print("\n| LayerNorm, H = 768 | rows | f32 + bf16 out µs | f32 + e4m3 out µs |")
    print("|---|---|---|---|")
    for rows in (3549, 12202):
        y = torch.randn(rows, 768, device="cuda").to(torch.bfloat16)
        res = torch.randn(rows, 768, device="cuda")
        gm, bt = torch.ones(768, device="cuda"), torch.zeros(768, device="cuda")
        t = alternate({"bf16": lambda: ops.layernorm(y, gm, bt, residual=res),
                       "e4m3": lambda: ops.layernorm_e4m3(y, gm, bt, residual=res)}, reps, iters)
        print(f"| | {rows} | {1e3 * t['bf16']:.1f} | {1e3 * t['e4m3']:.1f} |")


def bench_encoder(reps, iters):
    import _fp8_oracle as fo
    from oracle import nn as onn
    B, L = 64, 128
    cfg = dict(bert.BERT_BASE_CHINESE)
    store = variables.VariableStore("cuda", seed=11)
    bert.create_bert_variables(cfg, store)
    feats = synthetic.msra_batch(B, L, vocab=cfg["vocab_size"], seed=21)
    ids, mask, seg = (feats[k].cuda() for k in ("token_ids", "mask", "segment_ids"))
    pack = bert.make_pack(mask, int(feats["mask"].sum()))
    t = alternate({"bf16": lambda: bert.bert_forward(ids, mask, seg, cfg, store=store, pack=pack),
                   "fp8": lambda: bert.bert_forward_fp8(ids, mask, seg, cfg, store=store, pack=pack)}, reps, max(5, iters // 5))
    print(f"\n12-layer encoder, B = {B}, L = {L}, packed ({pack.total} tokens): bf16 {t['bf16']:.3f} ms = "
          f"{B / t['bf16'] * 1e3:.0f} sentences/s, fp8 {t['fp8']:.3f} ms = {B / t['fp8'] * 1e3:.0f} sentences/s "
          f"({t['bf16'] / t['fp8']:.2f}x)")
    w = store.state_dict()
    valid = (torch.arange(L)[None, :] < feats["seq_len"][:, None]).cuda()
    ref = onn.bert_encoder({k: v.cuda() for k, v in w.items() if k.startswith("bert/")}, ids, mask, seg, num_layers=12,
                           dtype=torch.float64)[valid]
    emu = fo.bert_encoder_fp8(w, feats["token_ids"], feats["mask"], feats["segment_ids"], num_layers=12, device="cuda")[valid]
    for name, fn in (("bf16", bert.bert_forward), ("fp8", bert.bert_forward_fp8)):
        x = fn(ids, mask, seg, cfg, store=store, pack=pack)[0].double()
        d = x - ref
        line = f"  {name}: vs float64 oracle max {d.abs().max().item():.3e}, rms {d.pow(2).mean().sqrt().item():.3e}"
        if name == "fp8":
            e = x - emu
            line += f"; vs fp8-emulated oracle max {e.abs().max().item():.3e}, rms {e.pow(2).mean().sqrt().item():.3e}"
        print(line)


def bench_plugins(reps, iters):
    B, L = 64, 128
    feats = synthetic.msra_batch(B, L, seed=5)
    print(f"\n| plugin PREDICT (build_graph path), B = {B}, L = {L} | bf16 sentences/s | fp8 sentences/s | fp8 speed-up |")
    print("|---|---|---|---|")
    for model_name in ("bert_bilstm_crf", "bert_crf"):
        est = engine.Estimator(model_name, dict(synthetic.data_params(L), pretrain_dir="", fused_predict=False))
        dev = est.to_device(feats)

        def run(prec):
            est.params["bert_precision"] = prec
            return est.predict_device(dev)
        t = alternate({"bf16": lambda: run("bf16"), "fp8": lambda: run("fp8")}, reps, max(5, iters // 5))
        print(f"| {model_name} | {B / t['bf16'] * 1e3:.0f} | {B / t['fp8'] * 1e3:.0f} | {t['bf16'] / t['fp8']:.2f}x |")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_fp8.py measures on the GPU"
    print("card (name, power limit, SM clock, max SM clock):", card())
    bench_gemms(args.reps, args.iters)
    bench_layernorm(args.reps, args.iters)
    bench_encoder(args.reps, args.iters)
    bench_plugins(args.reps, args.iters)
    print("card after the run:", card())


if __name__ == "__main__":
    main()
