"""Document mode on the GPU: the window plan, the stitch gathers, bert_bilstm_crf PREDICT on long documents, and a TRAIN
step at L = 2048.

usage: python scripts/bench_documents.py        (prints one JSON line)

  * ner_window_plan alone: B = 16 full-length documents of n = 4095 tokens, W = 512, S = 255.
  * the stitch of the packed PREDICT path: two ner_gather_rows launches (f32 and bf16 rows, H = 768) over B * n document
    rows; bytes count one read and one write of every row, given against the 3.35 TB/s HBM3 data-sheet figure.
  * PREDICT (Estimator.predict_device -> build_graph) of bert_bilstm_crf (BERT-base, 12 layers, random weights) for B = 16
    full-length documents at n = 1024, 2048 and 4095, with S = (W - 2) // 2 (the default) and S = W - 2 (no overlap:
    independent chunks, with the whole-document BiLSTM and CRF).  window_tokens / doc_tokens is the encoder's extra work.
  * TRAIN step (Estimator.train_step) of bert_bilstm_crf at B = 4, full-length L = 2048, default stride.
CUDA events over many calls; the card's name, power limit and max SM clock are read in the same run.
"""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from chinesener_b200 import engine, ops, synthetic, windows  # noqa: E402
from bench_long_seq import card, timeit  # noqa: E402

HBM_BPS = 3.35e12
W = 512


def bench_plan_and_stitch(B=16, n=4095, H=768):
    S = (W - 2) // 2
    feats = synthetic.msra_batch(B, n, seed=5, full=True)
    ids, seg, lens = (feats[k].cuda() for k in ("token_ids", "segment_ids", "seq_len"))
    NW, n_win = windows.window_counts(feats["seq_len"].numpy(), W, S)
    n_doc = int(feats["seq_len"].sum())
    plan_ms, plan_best = timeit(lambda: ops.window_plan(ids, seg, lens, W, S, NW, n_doc, packed=True), iters=50)
    src = ops.window_plan(ids, seg, lens, W, S, NW, n_doc, packed=True)["doc_src_packed"]
    x32 = torch.randn((n_win, H), device="cuda")
    x16 = x32.to(torch.bfloat16)
    st_ms, st_best = timeit(lambda: (ops.gather_rows(x32, src, n_doc), ops.gather_rows(x16, src, n_doc)), iters=50)
    nbytes = 2 * n_doc * H * (4 + 2)
    return dict(B=B, n=n, NW=NW, window_plan_us=plan_ms * 1e3, window_plan_best_us=plan_best * 1e3,
                stitch_us=st_ms * 1e3, stitch_best_us=st_best * 1e3, stitch_bytes=nbytes,
                stitch_share_of_3_35TBps=nbytes / (st_ms * 1e-3) / HBM_BPS)


def bench_predict(B=16, iters=10):
    out = {}
    for n in (1024, 2048, 4095):
        feats = synthetic.msra_batch(B, n, seed=7, full=True)
        for tag, S in (("half_overlap", (W - 2) // 2), ("no_overlap", W - 2)):
            est = engine.Estimator("bert_bilstm_crf", dict(synthetic.data_params(n), pretrain_dir="", bert_window=W,
                                                           bert_window_stride=S))
            dev = est.to_device(feats)
            est.predict_device(dev)                          # creates the variables
            ms, best = timeit(lambda: est.predict_device(dev), warm=2, iters=iters, spin=False)
            NW, n_win = windows.window_counts(feats["seq_len"].numpy(), W, S)
            doc_tokens = int(feats["mask"].sum())
            out[f"n{n}_{tag}"] = dict(S=S, windows=NW, window_tokens=n_win, doc_tokens=doc_tokens,
                                      encoder_token_factor=n_win / doc_tokens, predict_ms=ms, predict_best_ms=best,
                                      documents_per_s=B / ms * 1e3, tokens_per_s=doc_tokens / ms * 1e3)
            del est, dev
            torch.cuda.empty_cache()
    return out


def bench_train(B=4, L=2048, iters=6):
    feats = synthetic.msra_batch(B, L, seed=9, full=True)
    est = engine.Estimator("bert_bilstm_crf", dict(synthetic.data_params(L), pretrain_dir="", keep_prob_list=[0.9]))
    dev = est.to_device(feats)
    ms, best = timeit(lambda: est.train_step(dev), warm=2, iters=iters, spin=False)
    return dict(B=B, L=L, train_ms_per_step=ms, train_best_ms=best, tokens=int(feats["mask"].sum()))


def main():
    assert torch.cuda.is_available(), "bench_documents.py measures on a CUDA device"
    res = dict(card=card(), plan_and_stitch=bench_plan_and_stitch(), predict_B16=bench_predict(), train=bench_train())
    print(json.dumps(res))


if __name__ == "__main__":
    main()
