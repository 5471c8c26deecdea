"""GPU: TRAIN mode of the bert_crf plugin (BASELINE config 2's model) — the full encoder backward
(dense dgrad/wgrad on wgmma, attention backward, LayerNorm/GELU/embedding backward) against
autograd of the float64 oracle, and a short AdamW run."""
import json

import numpy as np
import pytest
import torch

from chinesener_b200 import autodiff, engine, synthetic, variables
from oracle import crf_torch, nn as onn

pytestmark = pytest.mark.gpu

CFG = {'vocab_size': 1500, 'hidden_size': 768, 'num_hidden_layers': 2, 'num_attention_heads': 12,
       'intermediate_size': 3072, 'max_position_embeddings': 128, 'type_vocab_size': 2, 'initializer_range': 0.02}


def _est(tmp_path, B=4, L=32, dropout=0.0, model="bert_crf", keep=1.0, bert_dropout=0.0):
    cfg = dict(CFG, hidden_dropout_prob=bert_dropout, attention_probs_dropout_prob=bert_dropout)
    (tmp_path / "bert_config.json").write_text(json.dumps(cfg))
    feats = synthetic.msra_batch(B, L, vocab=CFG['vocab_size'], seed=21)
    params = dict(synthetic.data_params(L), pretrain_dir=str(tmp_path), embedding_dropout=dropout, keep_prob_list=[keep])
    return engine.Estimator(model, params), feats


def _oracle(w, feats, lstm_activation=None):
    wd = {k: v.double().clone().requires_grad_(True) for k, v in w.items()}
    seq = onn.bert_encoder(wd, feats['token_ids'], feats['mask'], feats['segment_ids'], num_layers=2, num_heads=12,
                           dtype=torch.float64)
    if lstm_activation is not None:
        seq = onn.bilstm(seq, wd, feats['seq_len'], lstm_activation, 1.0, torch.float64)
    logits = seq @ wd['logits/kernel'] + wd['logits/bias']
    ll = crf_torch.crf_log_likelihood(logits, feats['label_ids'], feats['seq_len'], wd['crf_layer/transitions'])
    loss = (-ll).mean()
    loss.backward()
    return float(loss.detach()), {k: v.grad for k, v in wd.items()}


@pytest.mark.parametrize("per_kernel", [False, True, "packed"])
@pytest.mark.parametrize("model", ["bert_crf", "bert_bilstm_crf"])
def test_bert_gradients_match_oracle_autograd(tmp_path, model, per_kernel, monkeypatch):
    """bert_crf (config 2) and bert_bilstm_crf (the north-star plugin): d loss / d every variable, through the
    two-call C composite (ner_bert_encoder_train_fwd/_bwd) on the padded layout, through its sequence-packed form
    (…_packed: real tokens only) and through the one-call-per-kernel path."""
    from chinesener_b200 import bert as _bert
    from chinesener_b200.tools import layer as _layer
    monkeypatch.setattr(_layer, "TRAIN_PACK", per_kernel == "packed")
    per_kernel = per_kernel is True
    monkeypatch.setattr(_bert, "PER_KERNEL", per_kernel)
    est, feats = _est(tmp_path, model=model)
    est.evaluate(feats)
    est.store.vars["logits/kernel"].mul_(4.0)
    est.store.touch()
    w = est.store.state_dict()
    ref_loss, ref = _oracle(w, feats, est.params['rnn_activation'] if model == "bert_bilstm_crf" else None)
    dev = est.to_device(feats)
    with variables.use_store(est.store), autodiff.recording(est.store) as tape:
        loss, _ = est.build_graph(dev, None, est.params, True)
        tape.backward()
    assert abs(float(loss) - ref_loss) < 2e-2 * max(1.0, abs(ref_loss))
    worst = {}
    gscale = max(g.abs().max().item() for n, g in ref.items() if g is not None and "pooler" not in n)
    for name, g_ref in ref.items():
        if g_ref is None or "pooler" in name:
            continue
        g = est.store.grads[name].cpu().double()
        # key biases have an analytically ZERO gradient (softmax is shift-invariant along the keys), so
        # every variable is measured against max(its own scale, 1e-3 of the largest gradient)
        scale = max(g_ref.abs().max().item(), 1e-3 * gscale)
        worst[name] = (g - g_ref).abs().max().item() / scale
    bad = {k: v for k, v in worst.items() if v > 8e-2}
    print("max relative gradient error:", max(worst.values()), "over", len(worst), "variables")
    assert not bad, bad
    assert "bert/pooler/dense/kernel" not in est.store.grads      # unused by the reference: no gradient


@pytest.mark.parametrize("model", ["bert_crf", "bert_bilstm_crf"])
def test_bert_training_reduces_loss(tmp_path, model):
    est, feats = _est(tmp_path, dropout=0.1, model=model, keep=0.8, bert_dropout=0.1)   # every dropout site on
    # bert_bilstm_crf multiplies lr by 100 (lstm) / 500 (crf, logits) (diff_lr_times, reference
    # model/bert_bilstm_crf.py:45-47): its ReLU cells diverge at the lr bert_crf tolerates
    est.params.update(lr=2e-4 if model == "bert_crf" else 1e-5, num_train_steps=100, warmup_ratio=0.1)
    losses = [float(est.train_step(feats)) for _ in range(12)]
    print(model, "losses:", ["%.3f" % v for v in losses])
    assert np.isfinite(losses).all(), losses
    assert losses[-1] < 0.8 * losses[0], losses


def test_packed_and_padded_train_composites_agree(tmp_path, monkeypatch):
    """Same batch, dropout off: the packed composite's loss and every gradient equal the padded composite's up to the bf16
    GEMM summation order (the weight-gradient GEMMs run over K = real tokens instead of K = B*L)."""
    from chinesener_b200.tools import layer as _layer
    res = {}
    for packed in (False, True):
        monkeypatch.setattr(_layer, "TRAIN_PACK", packed)
        est, feats = _est(tmp_path, model="bert_bilstm_crf", B=6, L=48)
        dev = est.to_device(feats)
        with variables.use_store(est.store), autodiff.recording(est.store) as tape:
            loss, _ = est.build_graph(dev, None, est.params, True)
            tape.backward()
        res[packed] = (float(loss), {k: v.clone() for k, v in est.store.grads.items()})
    assert abs(res[True][0] - res[False][0]) < 2e-3 * max(1.0, abs(res[False][0]))
    gscale = max(float(g.abs().max()) for g in res[False][1].values())
    for name, g in res[False][1].items():
        scale = max(float(g.abs().max()), 1e-3 * gscale)
        assert float((res[True][1][name] - g).abs().max()) / scale < 3e-2, name


def test_row_gather_scatter_and_packed_attention_bwd():
    """ner_gather_rows / ner_scatter_rows are exact inverses on the packed rows; ner_bert_attention_bwd_packed equals the
    padded kernel on the real tokens (bf16 rounding tolerance 2e-2 of scale; the masked key tiles add exact zeros)."""
    from chinesener_b200 import ops
    g = torch.Generator().manual_seed(3)
    B, L, NH, D = 5, 48, 12, 64
    lens = torch.tensor([48, 1, 17, 33, 7])
    mask = (torch.arange(L)[None, :] < lens[:, None]).to(torch.int32).cuda()
    cu, tok_src = ops.seq_pack_plan(mask)
    n = int(lens.sum())
    x = torch.randn(B * L, 768, generator=g).cuda()
    xp = ops.gather_rows(x, tok_src, n)
    flat = torch.cat([torch.arange(int(l)) + b * L for b, l in enumerate(lens)])
    assert torch.equal(xp.cpu(), x.cpu()[flat])
    back = ops.scatter_rows(xp, tok_src, B * L).cpu()
    keep = torch.zeros(B * L, dtype=torch.bool)
    keep[flat] = True
    assert torch.equal(back[keep], x.cpu()[keep]) and float(back[~keep].abs().max()) == 0.0
    qkv = (torch.randn(B * L, 3 * NH * D, generator=g) * 0.5).to(torch.bfloat16).cuda()
    dctx = torch.randn(B * L, NH * D, generator=g).to(torch.bfloat16)
    dctx[~keep] = 0          # [PAD] queries carry no gradient in the model (in the padded kernel they would reach real keys)
    dctx = dctx.cuda()
    for keep_prob in (1.0, 0.9):
        ctx = ops.bert_attention(qkv, mask, B, L, NH, D, keep_prob=keep_prob, seed=77)
        dq = ops.bert_attention_bwd(qkv, mask, ctx, dctx, B, L, NH, D, keep_prob=keep_prob, seed=77)
        qp, cp, dp = (ops.gather_rows(t, tok_src, n) for t in (qkv, ctx, dctx))
        ctxp = ops.bert_attention(qp, None, B, L, NH, D, cu_seqlens=cu, keep_prob=keep_prob, seed=77)
        assert float((ctxp.float() - cp.float()).abs().max()) <= 1e-2 * float(cp.float().abs().max())
        dqp = ops.bert_attention_bwd(qp, None, cp, dp, B, L, NH, D, keep_prob=keep_prob, seed=77, cu_seqlens=cu)
        ref = ops.gather_rows(dq, tok_src, n)
        assert float((dqp.float() - ref.float()).abs().max()) <= 2e-2 * float(ref.float().abs().max())
