"""The bert_mrc_span plugin on the GPU: PREDICT and TRAIN against bert_mrc, and the span kernels alone.

usage: python scripts/bench_mrc_span.py        (prints one JSON line)

  * One B = 64, L = 128 MSRA-shaped batch (synthetic.msra_batch), BERT-base, random weights, bf16 encoder, T = 3 types with
    the default queries' lengths (bench_mrc.mrc_params).  predict: sentences/s of Estimator.predict_device; train: one
    Estimator.train_step (forward, backward, AdamW); CUDA events over many calls.
  * kernels: ner_mrc_span_match_fwd (fwd_keep1: keep 1, as in EVAL; fwd: keep 0.9 as in TRAIN; both with the loss),
    ner_mrc_span_match_bwd and ner_mrc_span_decode at
    I = 1024, full length (P = 192 pairs of 128 tokens) and MSRA-shaped (the batch's lengths, 3 pairs per sentence), each
    timed alone with CUDA events over launches queued behind a spin kernel.  The decode sees start / end logits that make
    about half of the positions starts and ends (what random weights give).  Rates are per candidate . k element of the
    match head (1 <= i <= j <= len - 2, k < I) and in FP32 FLOP/s by FLOPS_PER_ELEMENT, as a share of the H100 SXM
    data-sheet FP32 rate (67 TFLOP/s); the tanh is counted as no FLOP.
The card's name and power limit are read in the same run: a number is only meaningful next to them.
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from bench_mrc import card, mrc_params, timeit  # noqa: E402
from chinesener_b200 import engine, ops, synthetic  # noqa: E402

# FP32 FLOP per candidate . k element: forward x = u + v, x^2, c0 + c1 x^2 (fma), s = x (.), hx = x w/2, hx t + hx (fma),
# accumulate = 9; backward (dU pass: GELU', GELU and the dw2 term; dV pass: GELU') = 38
FLOPS_PER_ELEMENT = {'fwd_keep1': 9, 'fwd': 9, 'bwd': 38, 'decode': 9}
FP32_PEAK = 67e12


def bench_plugins(feats, B, L, iters_predict=50, iters_train=10):
    out = {}
    for name in ("bert_mrc_span", "bert_mrc"):
        est = engine.Estimator(name, mrc_params(L))
        est.evaluate(feats)                               # creates the variables
        dev = est.to_device(feats)
        ms, best = timeit(lambda: est.predict_device(dev), warm=5, iters=iters_predict, spin=False)
        tms, tbest = timeit(lambda: est.train_step(dev), warm=3, iters=iters_train, spin=False)
        out[name] = dict(predict_ms_per_batch=ms, predict_best_ms=best, sentences_per_s=B / ms * 1e3,
                         train_ms_per_step=tms, train_best_ms=tbest, last_loss=float(est.train_step(dev)))
        del est, dev
        torch.cuda.empty_cache()
    out["span_over_mrc_predict_time"] = out["bert_mrc_span"]["predict_ms_per_batch"] / out["bert_mrc"]["predict_ms_per_batch"]
    out["span_over_mrc_train_time"] = out["bert_mrc_span"]["train_ms_per_step"] / out["bert_mrc"]["train_ms_per_step"]
    return out


def bench_kernels(lens, T, L, I=1024, iters=20):
    P = len(lens)
    g = torch.Generator(device="cuda").manual_seed(5)
    uv = torch.randn((P * L, 2 * I), device="cuda", generator=g)
    b1 = 0.1 * torch.randn(I, device="cuda", generator=g)
    w2 = torch.randn(I, device="cuda", generator=g) / I ** 0.5
    b2 = torch.zeros(1, device="cuda")
    sl = torch.from_numpy(np.asarray(lens, np.int32)).cuda()
    labels = torch.randint(0, 3, (P, L), device="cuda", generator=g, dtype=torch.int32)
    span_end = ops.mrc_span_targets(labels, sl)[2]
    n_cand = int(sum(max(int(n) - 2, 0) * max(int(n) - 1, 0) // 2 for n in lens))
    z, _ = ops.mrc_span_match_fwd(uv, b1, w2, b2, sl, L, span_end, 0.9, 11)
    logits = torch.randn((P, L, 2), device="cuda", generator=g)
    sent_len = sl.view(-1, T)[:, 0].contiguous()
    tt = torch.tensor([[2 + 2 * t, 3 + 2 * t] for t in range(T)], dtype=torch.int32, device="cuda")
    runs = dict(fwd_keep1=lambda: ops.mrc_span_match_fwd(uv, b1, w2, b2, sl, L, span_end),
                fwd=lambda: ops.mrc_span_match_fwd(uv, b1, w2, b2, sl, L, span_end, 0.9, 11),
                bwd=lambda: ops.mrc_span_match_bwd(uv, z, b1, w2, sl, span_end, 1.0, 0.9, 11),
                decode=lambda: ops.mrc_span_decode(logits, logits.flip(-1).contiguous(), uv, b1, w2, b2, sent_len, tt, 1, 8, 9))
    out = dict(P=P, L=L, I=I, candidates=n_cand)
    for name, fn in runs.items():
        ms, best = timeit(fn, iters=iters)
        res = dict(us=ms * 1e3, best_us=best * 1e3)
        if name != "decode":                             # the decode evaluates starts x ends only: its element count varies
            el = n_cand * I
            res.update(elements_per_s=el / ms * 1e3, fp32_flops=el * FLOPS_PER_ELEMENT[name] / ms * 1e3)
            res["fp32_share"] = res["fp32_flops"] / FP32_PEAK
        out[name] = res
    return out


def main():
    assert torch.cuda.is_available(), "bench_mrc_span.py measures on a CUDA device"
    B, L, T = 64, 128, 3
    feats = synthetic.msra_batch(B, L, seed=1000)
    msra_lens = np.repeat(feats['seq_len'].numpy(), T)
    res = dict(card=card(), B=B, L=L, token_fill=float(feats["mask"].float().mean()),
               plugins=bench_plugins(feats, B, L),
               kernels_full=bench_kernels([L] * (B * T), T, L), kernels_msra=bench_kernels(msra_lens, T, L))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
