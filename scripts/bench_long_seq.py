"""Long sequences on the GPU: the attention backward on each side of the L = 384 switch, and bert_bilstm_crf at L = 512.

usage: python scripts/bench_long_seq.py        (prints one JSON line)

  * attention backward alone (ner_bert_attention_bwd, padded layout, every row full length): NH = 12, B * L ~ 32768
    tokens, L in {128, 256, 384} (one CTA per (sequence, head) holds the whole head) and {448, 512} (key-tiled kernels),
    keep_prob 1.0 and 0.9.  The algorithmic rate counts five L x L x 64 matmuls (S, dP, dV, dK, dQ) per (sequence, head)
    at 2 FLOP per multiply-add, whatever a kernel recomputes, and is given as a share of the 989 TFLOP/s dense BF16
    data-sheet figure.  ns per (query x key) pair compares the two kernels across the switch.
  * TRAIN step (Estimator.train_step) of bert_bilstm_crf (BERT-base, 12 layers, random weights) at B = 16: full-length
    L = 384, full-length L = 512, and MSRA-shaped lengths at L = 512.
  * PREDICT sentences/s (Estimator.predict_device, fused executor) of bert_bilstm_crf at L = 512, full-length and
    MSRA-shaped.
CUDA events over many calls; the card's name and power limit are read in the same run.
"""
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from chinesener_b200 import engine, ops, synthetic  # noqa: E402

PEAK_BF16 = 989e12
NH, D, TOKENS = 12, 64, 32768


def timeit(fn, warm=3, iters=20, spin=True):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    if spin:
        torch.cuda._sleep(8_000_000)
    for s, e in evs:
        s.record()
        fn()
        e.record()
    torch.cuda.synchronize()
    ts = sorted(s.elapsed_time(e) for s, e in evs)
    return ts[len(ts) // 2], ts[0]


def card():
    out = dict(name=torch.cuda.get_device_name(0))
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        out.update(power_limit_w=float(q[0]), max_sm_clock_mhz=float(q[1]))
    except Exception as e:          # the number is still reported, without the power limit
        out.update(power_limit_w=None, power_limit_error=repr(e))
    return out


def bench_attention_bwd(iters=30):
    g = torch.Generator(device="cuda").manual_seed(3)
    out = {}
    for L in (128, 256, 384, 448, 512):
        B = max(1, TOKENS // L)
        qkv = (torch.randn((B * L, 3 * NH * D), device="cuda", generator=g) * 0.7).to(torch.bfloat16)
        dctx = torch.randn((B * L, NH * D), device="cuda", generator=g).to(torch.bfloat16)
        mask = torch.ones((B, L), dtype=torch.int32, device="cuda")
        for keep in (1.0, 0.9):
            ctx = ops.bert_attention(qkv, mask, B, L, NH, D, keep_prob=keep, seed=11)
            ms, best = timeit(lambda: ops.bert_attention_bwd(qkv, mask, ctx, dctx, B, L, NH, D, keep_prob=keep, seed=11),
                              iters=iters)
            flop = 5 * 2 * B * NH * L * L * D
            pairs = B * NH * L * L
            out[f"L{L}_keep{keep}"] = dict(B=B, kernel="whole-head" if L <= 384 else "key-tiled", us=ms * 1e3, best_us=best * 1e3,
                                           tflops=flop / (ms * 1e-3) / 1e12, share_of_989=flop / (ms * 1e-3) / PEAK_BF16,
                                           ns_per_pair=ms * 1e6 / pairs)
        del qkv, dctx, ctx
    return out


def bench_models(B=16, predict_iters=20, train_iters=8):
    cases = [("full_L384", synthetic.msra_batch(B, 384, seed=7, full=True), 384),
             ("full_L512", synthetic.msra_batch(B, 512, seed=7, full=True), 512),
             ("msra_L512", synthetic.msra_batch(B, 512, seed=7), 512)]
    out = {}
    for name, feats, L in cases:
        est = engine.Estimator("bert_bilstm_crf", dict(synthetic.data_params(L), pretrain_dir="", keep_prob_list=[0.9]))
        est.evaluate(feats)                               # creates the variables
        dev = est.to_device(feats)
        t_ms, t_best = timeit(lambda: est.train_step(dev), warm=2, iters=train_iters, spin=False)
        res = dict(tokens=int(feats["mask"].sum()), train_ms_per_step=t_ms, train_best_ms=t_best)
        if L == 512:
            p_ms, p_best = timeit(lambda: est.predict_device(dev), warm=3, iters=predict_iters, spin=False)
            res.update(predict_sentences_per_s=B / p_ms * 1e3, predict_ms=p_ms, predict_best_ms=p_best)
        out[name] = res
        del est, dev
        torch.cuda.empty_cache()
    return out


def main():
    assert torch.cuda.is_available(), "bench_long_seq.py measures on a CUDA device"
    res = dict(card=card(), attention_bwd=bench_attention_bwd(), bert_bilstm_crf_B16=bench_models())
    print(json.dumps(res))


if __name__ == "__main__":
    main()
