"""Masked-LM pretraining on the GPU.

usage: python scripts/bench_mlm.py        (prints one JSON line)

  * ner_vocab_xent (loss + bf16 gradient + argmax) at M = 8192, V = 21128, ld = 21152: kernel time (median of CUDA
    events over the three launches), achieved bytes/s and its share of the 3.35 TB/s of the H100 SXM data sheet; the bytes
    are the V f32 logits read and the ld bf16 gradient elements written per row (4 V + 2 ld bytes);
  * ner_mlm_mask at B = 64, L = 128 and 512, with and without word_start;
  * the masked-LM TRAIN step (BERT-base-Chinese, max_predictions_per_seq 20, host batch included) against bert_crf's
    TRAIN step (Estimator.train_step) on the same MSRA-shaped B = 64, L = 128 batch, alternated over three rounds; and
    the head's share: the same step with the encoder replaced by a fixed output (masking, gather, transform, decoder,
    loss and the head's backward).
The card's name and power limit are read in the same run.
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from chinesener_b200 import autodiff, bert, engine, mlm, ops, pretrain, synthetic, variables  # noqa: E402
from chinesener_b200.tools import train_utils  # noqa: E402

HBM_BPS = 3.35e12


def bench_xent(iters=50):
    from bench_token_head import timeit
    M, V, ld = 8192, 21128, 21152
    g = torch.Generator().manual_seed(0)
    z = (torch.randn(M, ld, generator=g) * 3).cuda()
    y = torch.randint(0, V, (M,), generator=g, dtype=torch.int32).cuda()
    t = timeit(lambda: ops.vocab_xent(z, y, V, want_grad=True), warm=3, iters=iters)[0]
    nbytes = M * (4 * V + 2 * ld)
    return dict(M=M, V=V, ld=ld, us=t * 1e3, tb_s=nbytes / (t * 1e-3) / 1e12, share_of_hbm=nbytes / (t * 1e-3) / HBM_BPS)


def bench_mask(iters=200):
    from bench_token_head import timeit
    out = []
    for L in (128, 512):
        feats = synthetic.msra_batch(64, L, seed=1)
        n = feats['seq_len'].numpy()
        off = torch.from_numpy(mlm.pred_offsets(mlm.prediction_budget(n, 0.15, 20))).cuda()
        M = int(off[-1])
        ids, sl = feats['token_ids'].cuda(), feats['seq_len'].cuda()
        ws = (torch.rand(64, L) < 0.5).to(torch.uint8).cuda()
        for w in (None, ws):
            t = timeit(lambda: ops.mlm_mask(ids, sl, off, M, 7, 21128, 103, word_start=w), warm=3, iters=iters)[0]
            out.append(dict(B=64, L=L, word_start=w is not None, us=t * 1e3))
    return out


def mlm_step(cfg, store, feats):
    dev = pretrain.to_device(feats, torch.device('cuda'))
    store.dropout_calls = 0
    with variables.use_store(store), autodiff.recording(store) as tape:
        out = mlm.masked_lm(dev, cfg, store, store.global_step, 0.15, 20, 103, True, tape=tape)
        tape.backward()
        train_utils.bert_train_op(out.loss, 5e-5, 10000, 0.1, None, store=store)
    return out.loss


def head_only(cfg, store, feats, fixed):
    dev = pretrain.to_device(feats, torch.device('cuda'))
    keep = bert.bert_forward_train
    bert.bert_forward_train = lambda *a, **k: fixed
    try:
        with variables.use_store(store), autodiff.recording(store) as tape:
            out = mlm.masked_lm(dev, cfg, store, 5, 0.15, 20, 103, True, tape=tape)
            tape.backward()
    finally:
        bert.bert_forward_train = keep
    return out.loss


def bench_train(iters=20, rounds=3):
    from bench_token_head import timeit
    B, L = 64, 128
    feats = synthetic.msra_batch(B, L, seed=3)
    mfeats = {k: feats[k] for k in ('token_ids', 'mask', 'segment_ids', 'seq_len')}
    crf = engine.Estimator("bert_crf", dict(synthetic.data_params(L), pretrain_dir=''))
    cfg = bert.load_bert_config('')
    store = variables.VariableStore('cuda')
    fixed = torch.randn(B, L, cfg['hidden_size']).cuda()
    fixed.bf16 = fixed.to(torch.bfloat16)
    res = dict(B=B, L=L, crf_ms=[], mlm_ms=[], head_ms=[])
    for _ in range(rounds):
        res["crf_ms"].append(timeit(lambda: crf.train_step(feats), warm=3, iters=iters)[0])
        res["mlm_ms"].append(timeit(lambda: mlm_step(cfg, store, mfeats), warm=3, iters=iters)[0])
        res["head_ms"].append(timeit(lambda: head_only(cfg, store, mfeats, fixed), warm=3, iters=iters)[0])
    res["mlm_over_crf"] = float(np.median(res["mlm_ms"]) / np.median(res["crf_ms"]))
    res["head_share_of_mlm_step"] = float(np.median(res["head_ms"]) / np.median(res["mlm_ms"]))
    return res


def main():
    from bench_token_head import card
    out = dict(card=card())
    out["vocab_xent"] = bench_xent()
    out["mlm_mask"] = bench_mask()
    out["train_step"] = bench_train()
    out["aims"] = dict(mlm_step_le_1_15x_bert_crf=out["train_step"]["mlm_over_crf"] <= 1.15,
                       vocab_xent_ge_0_6_of_hbm=out["vocab_xent"]["share_of_hbm"] >= 0.6)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
