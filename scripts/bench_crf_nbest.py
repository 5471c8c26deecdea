"""N-best CRF decoding (ner_crf_viterbi_nbest) on the GPU.

usage: python scripts/bench_crf_nbest.py        (prints one JSON line)

  * kernel time (median of CUDA events) against ner_crf_viterbi at B = 64, L = 128, K = 10, for MSRA-shaped rows
    (synthetic.msra_batch lengths) and full-length rows, N in {1, 2, 4, 8, 16};
  * one large batch, B = 16384 full-length rows at N = 8, in sequences/s (against ner_crf_viterbi);
  * PREDICT sentences/s (Estimator.predict, host batch included) of bilstm_crf and bert_bilstm_crf on one MSRA-shaped
    B = 64 batch with crf_nbest 1 and 8; for 1, both the fused default and the layer path (crf_nbest > 1 decodes through
    build_graph, not the fused executor).
Every timed kernel output is checked against the numpy oracle (tests/_nbest_oracle.py) on a few rows first, and every
PREDICT output against the default run's pred_ids.  The card's name and power limit are read in the same run.
"""
import json
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tests"))
from chinesener_b200 import engine, ops, synthetic  # noqa: E402

import _nbest_oracle as nb  # noqa: E402

L, K = 128, 10


def make(B, msra, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, L, K, generator=g) * 2
    tr = torch.randn(K, K, generator=g) * 0.5
    lens = synthetic.msra_batch(B, L, seed=seed)['seq_len'].to(torch.int32) if msra else torch.full((B,), L, dtype=torch.int32)
    return x, tr, lens


def verify(x, tr, lens, N, got, rows):
    tags, scores, counts = (t.cpu().numpy() for t in got)
    rt, rs, rc = nb.nbest(x[rows].numpy(), tr.numpy(), lens[rows].numpy(), N)
    assert np.array_equal(tags[rows], rt) and np.array_equal(scores[rows].view(np.int32), rs.view(np.int32))
    assert np.array_equal(counts[rows], rc)


def bench_kernel(B, msra, Ns, iters):
    from bench_token_head import timeit
    x, tr, lens = make(B, msra)
    xd, trd, ld = x.cuda(), tr.cuda(), lens.cuda()
    t_vit = timeit(lambda: ops.crf_viterbi(xd, ld, trd, return_score=True), warm=5, iters=iters)[0]
    vt = ops.crf_viterbi(xd, ld, trd)
    rows = np.array([0, 1, B // 2, B - 1])
    out = dict(B=B, rows="msra" if msra else "full", viterbi_us=t_vit * 1e3,
               mean_len=float(lens.float().mean()), nbest={})
    for N in Ns:
        got = ops.crf_viterbi_nbest(xd, ld, trd, N)
        verify(x, tr, lens, N, got, rows)
        assert torch.equal(got[0][:, 0], vt)
        t = timeit(lambda: ops.crf_viterbi_nbest(xd, ld, trd, N), warm=5, iters=iters)[0]
        out["nbest"][N] = dict(us=t * 1e3, over_viterbi=t / t_vit, seq_per_s=B / (t * 1e-3))
    out["viterbi_seq_per_s"] = B / (t_vit * 1e-3)
    return out


def bench_predict(tmp, iters):
    from bench_token_head import timeit
    Bt = 64
    res = {}
    feats = synthetic.msra_batch(Bt, L, seed=3)
    for name in ("bilstm_crf", "bert_bilstm_crf"):
        if name.startswith("bert"):
            cfg = {'vocab_size': 21128, 'hidden_size': 768, 'num_hidden_layers': 12, 'num_attention_heads': 12,
                   'intermediate_size': 3072, 'max_position_embeddings': 512, 'type_vocab_size': 2,
                   'initializer_range': 0.02}
            with open(os.path.join(tmp, "bert_config.json"), "w") as f:
                json.dump(cfg, f)
            params = dict(synthetic.data_params(L), pretrain_dir=tmp)
        else:
            emb = torch.nn.functional.normalize(torch.randn(21128, 50), dim=1).numpy()
            params = dict(synthetic.data_params(L), embedding=emb)
        est = engine.Estimator(name, params)
        est.evaluate(feats)
        est.store.vars["logits/kernel"].mul_(8.0)
        est.store.touch()
        configs = [("n1_default", {}), ("n1_layer", {'fused_predict': False}), ("n8", {'crf_nbest': 8})]
        ref = est.predict(feats)['pred_ids']
        r = {}
        for label, extra in configs:
            saved = dict(est.params)
            est.params.update(extra)
            out = est.predict(feats)
            assert torch.equal(out['pred_ids'], ref), label
            if 'pred_nbest' in out:
                assert all(np.array_equal(p[0][0], ref[b].numpy()) for b, p in enumerate(out['pred_nbest']))
            t = timeit(lambda: est.predict(feats), warm=3, iters=iters)[0]
            r[label] = dict(ms=t, sentences_per_s=Bt / (t * 1e-3))
            est.params.clear()
            est.params.update(saved)
        r["n8_over_n1_layer"] = r["n8"]["sentences_per_s"] / r["n1_layer"]["sentences_per_s"]
        res[name] = r
    return res


def main():
    from bench_token_head import card
    out = dict(card=card(), L=L, K=K)
    Ns = [1, 2, 4, 8, 16]
    out["kernel_b64"] = [bench_kernel(64, True, Ns, 200), bench_kernel(64, False, Ns, 200)]
    out["kernel_b16384"] = bench_kernel(16384, False, [8], 20)
    with tempfile.TemporaryDirectory() as tmp:
        out["predict"] = bench_predict(tmp, 30)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
