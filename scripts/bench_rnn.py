"""The bidirectional RNN layer on the GPU: LSTM vs GRU cells, one vs two layers.

usage: python scripts/bench_rnn.py        (prints one JSON line)

  * kernels: ner_bilstm_recurrence / ner_bigru_recurrence (PREDICT form and TRAIN form with the saved tensors) and their
    BPTT kernels at B = 64, L = 128 with MSRA-shaped lengths (synthetic.msra_batch) and H in {128, 200}; CUDA events over
    many launches queued behind a spin kernel so the events bracket GPU work, not launch latency.
  * models: PREDICT sentences/s (Estimator.predict_device, device-resident features) and the TRAIN step
    (Estimator.train_step) of bilstm_crf and bert_bilstm_crf (BERT-base, random weights) for (lstm, 1), (gru, 1),
    (lstm, 2) and (gru, 2) layers of 128 units.  bert_bilstm_crf (lstm, 1) PREDICT runs the fused executor; the other
    settings run build_graph.
The card's name and power limit are read in the same run: a number is only meaningful next to them.
"""
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from chinesener_b200 import engine, ops, synthetic  # noqa: E402

SETTINGS = [("lstm", 1), ("gru", 1), ("lstm", 2), ("gru", 2)]


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


def bench_kernels(lens, B, L, iters=50):
    g = torch.Generator(device="cuda").manual_seed(5)
    sl = lens.cuda()
    out = {}
    for H in (128, 200):
        for cell, G in (("lstm", 4), ("gru", 3)):
            xproj = torch.randn((B * L, 2 * G * H), device="cuda", generator=g) * 0.5
            wf, wb = (torch.randn((H, G * H), device="cuda", generator=g) * H ** -0.5 for _ in range(2))
            d_out = torch.randn((B, L, 2 * H), device="cuda", generator=g)
            if cell == "lstm":
                fwd = lambda: ops.bilstm_recurrence(xproj, wf, wb, sl, B, L, H)
                saved = ops.bilstm_recurrence(xproj, wf, wb, sl, B, L, H, save_for_backward=True, keep_prob=0.8, seed=3)
                train = lambda: ops.bilstm_recurrence(xproj, wf, wb, sl, B, L, H, save_for_backward=True, keep_prob=0.8, seed=3)
                bwd = lambda: ops.bilstm_recurrence_bwd(d_out, saved[1], saved[2], wf, wb, sl, B, L, H, keep_prob=0.8, seed=3)
            else:
                fwd = lambda: ops.bigru_recurrence(xproj, wf, wb, sl, B, L, H)
                saved = ops.bigru_recurrence(xproj, wf, wb, sl, B, L, H, save_for_backward=True, keep_prob=0.8, seed=3)
                train = lambda: ops.bigru_recurrence(xproj, wf, wb, sl, B, L, H, save_for_backward=True, keep_prob=0.8, seed=3)
                bwd = lambda: ops.bigru_recurrence_bwd(d_out, saved[1], saved[2], wf, wb, sl, B, L, H, keep_prob=0.8, seed=3)
            res = {}
            for name, fn in (("fwd", fwd), ("fwd_train", train), ("bwd", bwd)):
                ms, best = timeit(fn, iters=iters)
                res[name] = dict(us=ms * 1e3, best_us=best * 1e3, us_per_step=ms * 1e3 / int(lens.max()))
            out[f"{cell}_H{H}"] = res
    return out


def bench_models(feats, B, L, predict_iters=30, train_iters=10):
    g = torch.Generator().manual_seed(0)
    char = torch.nn.functional.normalize(torch.randn(21128, 100, generator=g), dim=1).numpy()
    out = {}
    for model in ("bilstm_crf", "bert_bilstm_crf"):
        for cell, n in SETTINGS:
            rnn = dict(cell_type=cell, cell_size=n, hidden_units_list=[128] * n, keep_prob_list=[0.8] * n)
            params = dict(synthetic.data_params(L), **rnn)
            params.update(pretrain_dir="") if model.startswith("bert") else params.update(embedding=char)
            est = engine.Estimator(model, params)
            est.evaluate(feats)                               # creates the variables
            dev = est.to_device(feats)
            p_ms, p_best = timeit(lambda: est.predict_device(dev), warm=5, iters=predict_iters, spin=False)
            t_ms, t_best = timeit(lambda: est.train_step(dev), warm=3, iters=train_iters, spin=False)
            out[f"{model}_{cell}{n}"] = dict(predict_sentences_per_s=B / p_ms * 1e3, predict_ms=p_ms, predict_best_ms=p_best,
                                            train_ms_per_step=t_ms, train_best_ms=t_best)
            del est, dev
            torch.cuda.empty_cache()
    return out


def main():
    assert torch.cuda.is_available(), "bench_rnn.py measures on a CUDA device"
    B, L = 64, 128
    feats = synthetic.msra_batch(B, L, seed=1000)
    res = dict(card=card(), B=B, L=L, max_len=int(feats["seq_len"].max()), token_fill=float(feats["mask"].float().mean()),
               kernels=bench_kernels(feats["seq_len"], B, L), models=bench_models(feats, B, L))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
