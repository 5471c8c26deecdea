"""The bert_ce / bert_dice softmax heads on the GPU: ner_token_xent and ner_token_dice bandwidth, and bert_ce vs bert_crf
PREDICT throughput.

usage: python scripts/bench_token_head.py        (prints one JSON line)

  * kernel: B = 262144 sentences, L = 128, K = 10, MSRA-like lengths; PREDICT = argmax only, TRAIN = loss + d_logits +
    argmax in one call, TRAIN_DICE = the same with the Dice loss (ner_token_dice, the plugin's alpha = gamma = 1) on the
    same inputs and bytes.  GB/s = algorithmic bytes / median kernel time (CUDA events over many launches, queued behind a
    spin kernel so the events bracket GPU work, not launch latency).  Bytes per token: PREDICT 4K logits in + 4 pred_ids
    out; TRAIN 4K logits in + 4K d_logits out + 4 labels in + 4 pred_ids out (+ 4 per sentence for seq_len).  Every row
    of the outputs of both losses is checked against numpy (float64) outside the timed region.
  * model: sentences/s of Estimator.predict_device on one B = 64, L = 128 MSRA-shaped batch (synthetic.msra_batch), BERT
    base, random weights.  bert_ce runs the encoder on the padded layout (its [PAD] predictions are part of its output),
    bert_crf on the packed one.
The card's name and power limit are read in the same run: a number is only meaningful next to them.
"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from chinesener_b200 import engine, ops, synthetic  # noqa: E402


def timeit(fn, warm=3, iters=20):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
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


def check_rows(z, labels, lens, pred, loss, dz, chunk=8192):
    """Every row: pred == np.argmax (bit-exact), d_logits vs float64 within 1e-6, loss vs float64 within 1e-5 relative."""
    B, L, K = z.shape
    n = int(np.clip(lens, 0, L).sum())
    total, worst = 0.0, 0.0
    assert np.array_equal(pred, np.argmax(z, axis=-1).astype(np.int32)), "pred_ids differ from np.argmax"
    for s in range(0, B, chunk):
        zc = z[s:s + chunk].astype(np.float64)
        m = zc.max(-1, keepdims=True)
        e = np.exp(zc - m)
        se = e.sum(-1, keepdims=True)
        lse = (m + np.log(se))[..., 0]
        y = labels[s:s + chunk]
        valid = np.arange(L)[None, :] < lens[s:s + chunk, None]
        ce = lse - np.take_along_axis(zc, y[..., None].astype(np.int64), -1)[..., 0]
        total += float(ce[valid].sum())
        g = (e / se - np.eye(K)[y]) / n
        g[~valid] = 0.0
        worst = max(worst, float(np.abs(dz[s:s + chunk] - g).max()))
    ref = total / n
    assert abs(loss - ref) <= 1e-5 * abs(ref), (loss, ref)
    assert worst < 1e-6, worst
    return dict(loss=loss, loss_ref=ref, max_abs_dlogits_err=worst)


def check_rows_dice(z, labels, lens, pred, loss, dz, alpha, gamma, chunk=2048):
    """Every row of ner_token_dice: pred == np.argmax (bit-exact), loss vs float64 within 1e-5 relative, d_logits vs the
    float64 closed-form gradient within 1e-5 of its largest magnitude."""
    B, L, K = z.shape
    n = int(np.clip(lens, 0, L).sum())
    total, worst, gmax = 0.0, 0.0, 0.0
    assert np.array_equal(pred, np.argmax(z, axis=-1).astype(np.int32)), "pred_ids differ from np.argmax"
    for s in range(0, B, chunk):
        zc = z[s:s + chunk].astype(np.float64)
        e = np.exp(zc - zc.max(-1, keepdims=True))
        se = e.sum(-1, keepdims=True)
        top = np.eye(K, dtype=bool)[np.argmax(zc, -1)]
        sm = np.where(top, np.where(top, 0.0, e).sum(-1, keepdims=True), se - e)      # sum_{i != k} e_i
        p, u = e / se, sm / se
        ua = u ** alpha
        q = ua * p
        oh = np.eye(K, dtype=bool)[labels[s:s + chunk]]
        inv = 1.0 / (q + np.where(oh, 1.0 + gamma, gamma))
        c = np.where(oh, -(2.0 + gamma), gamma) * inv * inv * p * ua * (u - alpha * p)
        r = np.divide(c, sm, out=np.zeros_like(c), where=sm > 0)
        g = (c - e * (r.sum(-1, keepdims=True) - r)) / n
        valid = np.arange(L)[None, :] < lens[s:s + chunk, None]
        total += float((np.where(oh, 1.0 - q, q) * inv).sum(-1)[valid].sum())
        g[~valid] = 0.0
        worst = max(worst, float(np.abs(dz[s:s + chunk] - g).max()))
        gmax = max(gmax, float(np.abs(g).max()))
    ref = total / n
    assert abs(loss - ref) <= 1e-5 * abs(ref), (loss, ref)
    assert worst <= 1e-5 * gmax, (worst, gmax)
    return dict(loss=loss, loss_ref=ref, max_abs_dlogits_err=worst, max_abs_dlogits=gmax)


def bench_kernel(B=262144, L=128, K=10):
    g = torch.Generator(device="cuda").manual_seed(1234)
    z = torch.randn(B, L, K, device="cuda", generator=g) * 3.0
    labels = torch.randint(0, K, (B, L), device="cuda", dtype=torch.int32, generator=g)
    lens = torch.from_numpy(synthetic.msra_lengths(B, L, np.random.default_rng(7), False).astype(np.int32)).cuda()
    pred_ms, pred_best = timeit(lambda: ops.token_xent(z))
    train_ms, train_best = timeit(lambda: ops.token_xent(z, labels, lens, want_grad=True))
    dice_ms, dice_best = timeit(lambda: ops.token_dice(z, labels, lens, 1.0, 1.0, want_grad=True))
    pred, loss, dz = ops.token_xent(z, labels, lens, want_grad=True)
    pred_only = ops.token_xent(z)[0]
    torch.cuda.synchronize()
    assert torch.equal(pred, pred_only)
    zh, yh, nh = z.cpu().numpy(), labels.cpu().numpy(), lens.cpu().numpy()
    checked = check_rows(zh, yh, nh, pred.cpu().numpy(), float(loss), dz.cpu().numpy())
    del dz
    pred, loss, dz = ops.token_dice(z, labels, lens, 1.0, 1.0, want_grad=True)
    checked_dice = check_rows_dice(zh, yh, nh, pred.cpu().numpy(), float(loss), dz.cpu().numpy(), 1.0, 1.0)
    tokens = B * L
    pb, tb = tokens * (4 * K + 4), tokens * (8 * K + 8) + 4 * B
    return dict(B=B, L=L, K=K, fill=float(lens.float().mean()) / L,
                predict=dict(ms=pred_ms, best_ms=pred_best, bytes=pb, GBps=pb / pred_ms / 1e6),
                train=dict(ms=train_ms, best_ms=train_best, bytes=tb, GBps=tb / train_ms / 1e6),
                train_dice=dict(ms=dice_ms, best_ms=dice_best, bytes=tb, GBps=tb / dice_ms / 1e6,
                                over_train=dice_ms / train_ms),
                check=checked, check_dice=checked_dice)


def bench_models(B=64, L=128, iters=50):
    feats = synthetic.msra_batch(B, L, seed=1000)
    out = {}
    for name in ("bert_ce", "bert_crf"):
        est = engine.Estimator(name, dict(synthetic.data_params(L), pretrain_dir=""))
        est.evaluate(feats)                               # creates the variables
        dev = est.to_device(feats)
        ms, best = timeit(lambda: est.predict_device(dev), warm=5, iters=iters)
        out[name] = dict(ms_per_batch=ms, best_ms=best, sentences_per_s=B / ms * 1e3)
        del est
        torch.cuda.empty_cache()
    out["bert_ce_over_bert_crf_time"] = out["bert_ce"]["ms_per_batch"] / out["bert_crf"]["ms_per_batch"]
    out["token_fill"] = float(feats["mask"].float().mean())
    return dict(B=B, L=L, **out)


def main():
    assert torch.cuda.is_available(), "bench_token_head.py measures on a CUDA device"
    res = dict(card=card(), kernel=bench_kernel(), predict=bench_models())
    print(json.dumps(res))


if __name__ == "__main__":
    main()
