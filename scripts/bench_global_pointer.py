"""The bert_global_pointer plugin on the GPU: PREDICT and TRAIN against bert_crf and bert_mrc_span, and the GlobalPointer
kernels alone.

usage: python scripts/bench_global_pointer.py        (prints one JSON line)

  * plugins: one B = 64, L = 128 MSRA-shaped batch (synthetic.msra_batch), BERT-base, random weights, bf16 encoder, T = 3.
    predict: sentences/s of Estimator.predict_device; train: one Estimator.train_step (forward, backward, AdamW); CUDA
    events over many calls.
  * kernels: ner_gp_loss_fwd (bf16 and split), ner_gp_loss_bwd and ner_gp_decode at B = 16, T = 10, L = 512 full length
    (CLUENER-sized) and on the MSRA-shaped batch (B = 64, T = 3, L = 128, the batch's lengths), each timed alone with CUDA
    events over launches queued behind a spin kernel.  Rates are per candidate element (b, t, i, j with
    1 <= i <= j <= len - 2), in TFLOP/s counting 2 D FLOP per element for the forward and 6 D for the backward (D = 64),
    and as a share of the bound that applies: the forward's one exponential per element against the MUFU rate
    132 SMs x 16 / clk x 1.98 GHz = 4.2e12 / s (computed from the clock, not measured), the backward's FLOPs against the
    data-sheet dense BF16 rate (989 TFLOP/s).
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

D = ops.GP_HEAD
MUFU_BOUND = 132 * 16 * 1.98e9          # exponentials / s
BF16_PEAK = 989e12


def bench_plugins(feats, B, L, iters_predict=50, iters_train=10):
    out = {}
    for name in ("bert_global_pointer", "bert_crf", "bert_mrc_span"):
        params = mrc_params(L) if name == "bert_mrc_span" else dict(synthetic.data_params(L), pretrain_dir="")
        est = engine.Estimator(name, params)
        est.evaluate(feats)                               # creates the variables
        dev = est.to_device(feats)
        ms, best = timeit(lambda: est.predict_device(dev), warm=5, iters=iters_predict, spin=False)
        tms, tbest = timeit(lambda: est.train_step(dev), warm=3, iters=iters_train, spin=False)
        out[name] = dict(predict_ms_per_batch=ms, predict_best_ms=best, sentences_per_s=B / ms * 1e3,
                         train_ms_per_step=tms, train_best_ms=tbest, last_loss=float(est.train_step(dev)))
        del est, dev
        torch.cuda.empty_cache()
    gp_, crf, span = out["bert_global_pointer"], out["bert_crf"], out["bert_mrc_span"]
    out["gp_over_crf_predict_rate"] = gp_["sentences_per_s"] / crf["sentences_per_s"]
    out["gp_over_mrc_span_predict_rate"] = gp_["sentences_per_s"] / span["sentences_per_s"]
    out["gp_over_crf_train_time"] = gp_["train_ms_per_step"] / crf["train_ms_per_step"]
    return out


def bench_kernels(lens, T, L, iters=20):
    B = len(lens)
    g = torch.Generator(device="cuda").manual_seed(5)
    proj = torch.randn((B * L, T * 2 * D), device="cuda", generator=g)
    sl = torch.from_numpy(np.asarray(lens, np.int32)).cuda()
    labels = torch.randint(1, 2 + 2 * T, (B, L), device="cuda", generator=g, dtype=torch.int32)
    tt = torch.tensor([[2 + 2 * t, 3 + 2 * t] for t in range(T)], dtype=torch.int32, device="cuda")
    span_end = ops.gp_targets(labels, sl, tt)
    hi, lo = ops.gp_rope(proj, B, L, T, split=True)
    _, lse = ops.gp_loss_fwd(hi, None, sl, span_end, L)
    n_cand = T * int(sum(max(int(n) - 2, 0) * max(int(n) - 1, 0) // 2 for n in lens))
    runs = dict(loss_fwd=lambda: ops.gp_loss_fwd(hi, None, sl, span_end, L),
                loss_fwd_split=lambda: ops.gp_loss_fwd(hi, lo, sl, span_end, L),
                loss_bwd=lambda: ops.gp_loss_bwd(hi, sl, span_end, lse, L),
                rope=lambda: ops.gp_rope(proj, B, L, T),
                decode=lambda: ops.gp_decode(hi, None, sl, tt, 1, 8, 9, L))
    out = dict(B=B, T=T, L=L, candidates=n_cand)
    for name, fn in runs.items():
        ms, best = timeit(fn, iters=iters)
        res = dict(us=ms * 1e3, best_us=best * 1e3, elements_per_s=n_cand / ms * 1e3)
        if name.startswith("loss_fwd"):
            res["tflops"] = n_cand * 2 * D * (3 if name.endswith("split") else 1) / ms * 1e3 / 1e12
            res["mufu_share"] = res["elements_per_s"] / MUFU_BOUND
        elif name == "loss_bwd":
            res["tflops"] = n_cand * 6 * D / ms * 1e3 / 1e12
            res["bf16_share"] = res["tflops"] * 1e12 / BF16_PEAK
        out[name] = res
    return out


def main():
    assert torch.cuda.is_available(), "bench_global_pointer.py measures on a CUDA device"
    B, L, T = 64, 128, 3
    feats = synthetic.msra_batch(B, L, seed=1000)
    res = dict(card=card(), B=B, L=L, token_fill=float(feats["mask"].float().mean()),
               kernels_cluener=bench_kernels([512] * 16, 10, 512),
               kernels_msra=bench_kernels(feats['seq_len'].numpy(), T, L),
               plugins=bench_plugins(feats, B, L))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
