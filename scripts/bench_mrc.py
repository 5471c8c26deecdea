"""The bert_mrc plugin on the GPU: PREDICT throughput against bert_crf, the TRAIN step, and the two MRC kernels.

usage: python scripts/bench_mrc.py        (prints one JSON line)

  * One B = 64, L = 128 MSRA-shaped batch (synthetic.msra_batch), BERT-base, random weights, bf16 encoder.  bert_mrc runs
    T = 3 entity types (ORG, PER, LOC) with queries of the default queries' lengths (22, 10 and 20 tokens; random ids,
    synthetic mode has no vocabulary), so its packed encoder sees T * tokens + 55 * sentences rows against bert_crf's
    tokens.
  * predict: sentences/s of Estimator.predict_device (device-resident features, CUDA events over many calls).
  * train: one bert_mrc Estimator.train_step (forward, backward, AdamW), CUDA events.
  * kernels: ner_mrc_pairs on the batch and ner_mrc_merge on its [B*T, L, 3] logits, CUDA events over many launches
    queued behind a spin kernel so the events bracket GPU work, not launch latency.
The card's name and power limit are read in the same run: a number is only meaningful next to them.
"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from chinesener_b200 import _lib, engine, ops, synthetic  # noqa: E402
from chinesener_b200.data import mrc  # noqa: E402

QUERY_LENS = {'ORG': 22, 'PER': 10, 'LOC': 20}


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


def mrc_params(L):
    rng = np.random.default_rng(7)
    ids = {n: rng.integers(106, 21128, size=k).tolist() for n, k in QUERY_LENS.items()}
    return dict(synthetic.data_params(L), pretrain_dir="", mrc_query_ids=ids)


def bench_predict(feats, B, L, iters=50):
    out = {}
    for name in ("bert_mrc", "bert_crf"):
        params = mrc_params(L) if name == "bert_mrc" else dict(synthetic.data_params(L), pretrain_dir="")
        est = engine.Estimator(name, params)
        est.evaluate(feats)                               # creates the variables
        dev = est.to_device(feats)
        ms, best = timeit(lambda: est.predict_device(dev), warm=5, iters=iters, spin=False)
        out[name] = dict(ms_per_batch=ms, best_ms=best, sentences_per_s=B / ms * 1e3)
        if name == "bert_mrc":
            table = mrc.device_table(est.params)
            out[name]["encoder_rows"] = table.pair_tokens(dev['mask'])
        else:
            out[name]["encoder_rows"] = dev['mask'].total_tokens
        del est, dev
        torch.cuda.empty_cache()
    out["bert_mrc_over_bert_crf_time"] = out["bert_mrc"]["ms_per_batch"] / out["bert_crf"]["ms_per_batch"]
    return out


def bench_train(feats, L, iters=10):
    est = engine.Estimator("bert_mrc", mrc_params(L))
    dev = est.to_device(feats)
    ms, best = timeit(lambda: est.train_step(dev), warm=3, iters=iters, spin=False)
    loss = float(est.train_step(dev))
    del est
    torch.cuda.empty_cache()
    return dict(ms_per_step=ms, best_ms=best, last_loss=loss)


def bench_kernels(feats, L, iters=200):
    params = mrc_params(L)
    table = mrc.MrcTable(params)
    dev = {k: v.cuda() for k, v in feats.items()}
    B = dev['token_ids'].shape[0]
    BT = B * table.T
    # outputs allocated once and the library called directly: the timed launches are not paced by host allocations
    out = ops.mrc_pairs(dev['token_ids'], dev['seq_len'], table.query_ids, table.query_len, table.type_tag, table.L2,
                        table.sep_id, label_ids=dev['label_ids'])
    logits = torch.randn((BT, L, 3), device="cuda", generator=torch.Generator(device="cuda").manual_seed(3))
    pred = torch.empty((B, L), dtype=torch.int32, device="cuda")
    h, p = _lib.lib(), _lib.ptr
    pairs = lambda: _lib.check(h.ner_mrc_pairs(
        p(dev['token_ids']), p(dev['seq_len']), p(dev['label_ids']), p(table.query_ids), p(table.query_len), p(table.type_tag),
        B, L, table.T, table.qmax, table.L2, table.sep_id, p(out['ids']), p(out['segment_ids']), p(out['mask']),
        p(out['seq_len']), p(out['labels']), p(out['align']), _lib.stream()))
    merge = lambda: _lib.check(h.ner_mrc_merge(p(logits), p(dev['seq_len']), p(table.type_tag), B, L, table.T, table.o_tag,
                                               table.cls_tag, table.sep_tag, p(pred), _lib.stream()))
    pairs_ms, pairs_best = timeit(pairs, iters=iters)
    merge_ms, merge_best = timeit(merge, iters=iters)
    assert torch.equal(pred, ops.mrc_merge(logits, dev['seq_len'], table.type_tag, table.o_tag, table.cls_tag, table.sep_tag))
    pairs_bytes = 4 * (3 * BT * table.L2 + 2 * BT * L + BT) + 4 * 2 * B * L      # outputs + token / label reads
    merge_bytes = 4 * (BT * L * 3 + B * L)
    return dict(T=table.T, L2=table.L2,
                mrc_pairs=dict(us=pairs_ms * 1e3, best_us=pairs_best * 1e3, bytes=pairs_bytes, GBps=pairs_bytes / pairs_ms / 1e6),
                mrc_merge=dict(us=merge_ms * 1e3, best_us=merge_best * 1e3, bytes=merge_bytes, GBps=merge_bytes / merge_ms / 1e6))


def main():
    assert torch.cuda.is_available(), "bench_mrc.py measures on a CUDA device"
    B, L = 64, 128
    feats = synthetic.msra_batch(B, L, seed=1000)
    res = dict(card=card(), B=B, L=L, token_fill=float(feats["mask"].float().mean()),
               predict=bench_predict(feats, B, L), train=bench_train(feats, L), kernels=bench_kernels(feats, L))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
