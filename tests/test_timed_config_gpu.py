"""GPU parity at the configurations bench.py TIMES — 12-layer BERT-base-Chinese, full batch sizes.

  config 3 (BASELINE configs[2], the headline): bert_bilstm_crf, B=64, L=128, MSRA-shaped lengths, bf16 operands,
      through Estimator.predict_iter(streams=4) (the e2e path), blocking Estimator.predict (the fused one-call step)
      and build_graph; emission logits vs the oracle with the same bf16 rounding points and vs the float64 oracle;
      Viterbi bit-exact on the CUDA logits; tag agreement with the end-to-end oracle reported as a number.
  config 2 (BASELINE configs[1]): bert_crf, B=32, L=128, params['bert_precision']='fp32': emission logits within the
      north-star 1e-3 of the float64 oracle at 12 layers.

Parity is "unpinned" in the sense of SURVEY 8(c): no reference artefact holds logits; the oracle restates TF 1.14 /
bert-base 0.0.9 semantics and is itself checked against HuggingFace BertModel / torch.nn.LSTM / brute force.
Tolerances are written at each assert.  The measured errors are printed (pytest -s).
"""
import json

import numpy as np
import pytest
import torch

from chinesener_b200 import engine, synthetic, variables
from chinesener_b200.config import BERT_BASE_CHINESE
from oracle import crf, models as omodels

pytestmark = pytest.mark.gpu


def _estimator(model_name, tmp_path, L, **extra):
    (tmp_path / "bert_config.json").write_text(json.dumps(BERT_BASE_CHINESE))
    params = dict(synthetic.data_params(L), pretrain_dir=str(tmp_path), **extra)
    return engine.Estimator(model_name, params)


def _cuda_logits(est, dev, model_name, precision='bf16'):
    from chinesener_b200.tools import layer
    prec0, layer.BERT_PRECISION = layer.BERT_PRECISION, precision
    try:
        with variables.use_store(est.store):
            emb = layer.pretrain_bert_embedding(dev['token_ids'], dev['mask'], dev['segment_ids'], est.params['pretrain_dir'], 0.1, False)
            if model_name == "bert_bilstm_crf":
                emb = layer.bilstm(emb, 'lstm', est.params['rnn_activation'], [128], [1.0], 1, dev['seq_len'], 'float32', False)
            return layer.dense(emb, 10, 'logits')
    finally:
        layer.BERT_PRECISION = prec0


def test_config3_bert_bilstm_crf_b64_l128_12_layers(tmp_path):
    B, L = 64, 128
    est = _estimator("bert_bilstm_crf", tmp_path, L)
    batches = [synthetic.msra_batch(B, L, seed=1234 + i) for i in range(5)]           # bench.py's host batches
    est.evaluate(batches[0])                                                        # creates the variables
    est.store.vars["logits/kernel"].mul_(8.0)                                       # emissions O(1): non-trivial Viterbi paths
    est.store.touch()
    feats = batches[0]
    dev = est.to_device(feats)
    w = est.store.state_dict()
    trans = w['crf_layer/transitions'].numpy()
    lens = feats['seq_len'].numpy()
    valid = torch.arange(L)[None, :] < feats['seq_len'][:, None]

    # --- the three PREDICT routes agree
    pred_graph = est.forward_device(dev, False)[1].cpu().numpy()                    # build_graph, layer by layer
    pred_fused = est.predict(feats)['pred_ids'].numpy()                             # one-call step (fastpath), blocking
    outs = list(est.predict_iter(iter(batches), depth=5, streams=4))                # the e2e path of bench.py
    pred_iter = outs[0]['pred_ids'].numpy()
    assert pred_fused.dtype == np.int32 and pred_fused.shape == (B, L)
    np.testing.assert_array_equal(pred_fused, pred_graph)
    # 4 streams switch the GEMM tile policy (128x256 tiles): same K order per output element -> same bits expected;
    # a differing tag would have to come from an fp32 re-association, so the bar is equality on >= 99.9 % of tags
    agree_iter = float((pred_iter == pred_fused).mean())
    print(f"config 3: predict_iter(streams=4) vs blocking predict: {agree_iter:.6f} of tags equal")
    assert agree_iter >= 0.999
    for i, o in enumerate(outs[1:], 1):                                             # every batch of the stream pipeline
        ref_i = est.predict(batches[i])['pred_ids'].numpy()
        assert float((o['pred_ids'].numpy() == ref_i).mean()) >= 0.999
    assert (pred_fused[~valid.numpy()] == 0).all()                                  # zero beyond seq_len (tools/layer.py:147)
    # stacked calls (bench.py's second pipeline: `group` host batches per PREDICT call): sentences are independent, so the
    # tags are those of the separate calls (5 batches, group 4 -> one call of 4 and one of 1; group 8 -> one call of 5)
    for streams, group in ((2, 4), (2, 8)):
        outs_g = list(est.predict_iter(iter(batches), depth=3, streams=streams, group=group))
        assert len(outs_g) == len(batches)
        for i, o in enumerate(outs_g):
            ref_i = est.predict(batches[i])['pred_ids'].numpy()
            assert o['pred_ids'].shape == ref_i.shape
            assert float((o['pred_ids'].numpy() == ref_i).mean()) >= 0.999, (streams, group, i)

    # --- emission logits of the CUDA path vs the oracle
    logits = _cuda_logits(est, dev, "bert_bilstm_crf").cpu()
    p = dict(est.params, num_hidden_layers=12, num_attention_heads=12)
    ref_emul = omodels.bert_bilstm_crf(w, feats, p, dtype=torch.float64, emulate_bf16=True)
    ref_true = omodels.bert_bilstm_crf(w, feats, p, dtype=torch.float64, emulate_bf16=False)
    scale = ref_true['logits'][valid].abs().max().item()
    err_emul = (logits.double() - ref_emul['logits'])[valid].abs().max().item()
    err_true = (logits.double() - ref_true['logits'])[valid].abs().max().item()
    rms_true = (logits.double() - ref_true['logits'])[valid].pow(2).mean().sqrt().item()
    print(f"config 3 (12 layers, B=64, L=128, bf16 operands): max|logit - oracle(bf16 rounding points)| = {err_emul:.3e}, "
          f"max|logit - fp64 oracle| = {err_true:.3e} (rms {rms_true:.3e}), max|logit| = {scale:.2f}")
    # bf16 operands: a rounding flip moves one 768-term dot product by ~2^-9 relative; 12 layers of them.  The bar vs
    # the same-rounding oracle is 1e-2 of the logit scale, vs exact arithmetic 1e-1 of it (bf16 has 8 mantissa bits;
    # the north star's 1e-3 is the fp32 configuration's bar, tested below on config 2)
    assert err_emul < 1e-2 * max(1.0, scale)
    assert err_true < 1e-1 * max(1.0, scale)

    # --- Viterbi: bit-exact on the CUDA path's own fp32 logits (tags AND the zero fill)
    ref_pred, _ = crf.crf_decode(logits.numpy(), trans, lens, dtype=np.float32)
    np.testing.assert_array_equal(pred_graph, ref_pred)
    # --- and the end-to-end oracles (their own logits) as a rate
    agree_emul = float((pred_graph == ref_emul['pred_ids'])[valid.numpy()].mean())
    agree_true = float((pred_graph == ref_true['pred_ids'])[valid.numpy()].mean())
    print(f"config 3: tag agreement with the end-to-end oracle: {agree_emul:.5f} (bf16 rounding points), {agree_true:.5f} (fp64)")
    assert agree_emul >= 0.99 and agree_true >= 0.97
    # --- EVAL loss on the CUDA logits
    ll_ref = crf.crf_log_likelihood(logits.numpy(), feats['label_ids'].numpy(), lens, trans)
    loss = est.evaluate(feats)['loss']
    assert abs(loss - float(np.mean(-ll_ref))) < 1e-3 * max(1.0, abs(loss))


def test_config2_bert_crf_fp32_b32_l128_12_layers(tmp_path):
    B, L = 32, 128
    est = _estimator("bert_crf", tmp_path, L, bert_precision='fp32')
    feats = synthetic.msra_batch(B, L, seed=4321)
    est.evaluate(feats)
    est.store.vars["logits/kernel"].mul_(8.0)
    est.store.touch()
    out = est.evaluate(feats)
    w = est.store.state_dict()
    p = dict(est.params, num_hidden_layers=12, num_attention_heads=12)
    ref = omodels.bert_crf(w, feats, p, dtype=torch.float64, emulate_bf16=False)
    dev = est.to_device(feats)
    logits = _cuda_logits(est, dev, "bert_crf", precision='fp32').cpu()
    valid = torch.arange(L)[None, :] < feats['seq_len'][:, None]
    err = (logits.double() - ref['logits'])[valid].abs().max().item()
    scale = ref['logits'][valid].abs().max().item()
    print(f"config 2 (12 layers, B=32, L=128, fp32 mode): max|logit - fp64 oracle| = {err:.3e} (max |logit| {scale:.2f})")
    assert err < 1e-3                                      # the north-star tolerance for fp32 emission logits, absolute
    assert abs(out['loss'] - ref['loss']) < 1e-3 * max(1.0, abs(ref['loss']))
    ref_pred, _ = crf.crf_decode(logits.numpy(), w['crf_layer/transitions'].numpy(), feats['seq_len'].numpy(), dtype=np.float32)
    np.testing.assert_array_equal(out['pred_ids'].numpy(), ref_pred)       # Viterbi bit-exact on the CUDA logits
    agree = float((out['pred_ids'].numpy() == ref['pred_ids'])[valid.numpy()].mean())
    print(f"config 2: tag agreement with the fp64 end-to-end oracle: {agree:.5f}")
    assert agree >= 0.999
    # Estimator.predict (the public PREDICT call) runs the same fp32-accurate encoder
    np.testing.assert_array_equal(est.predict(feats)['pred_ids'].numpy(), out['pred_ids'].numpy())
