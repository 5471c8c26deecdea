"""GPU: training and inference on sequences longer than 384 tokens, up to BERT's 512 positions.

The attention backward stages a whole head in shared memory up to L = 384; longer sequences take the key-tiled kernels
(row statistics, dK/dV, dQ).  Checked here:
  * the tiled backward against float64 autograd, padded and packed, with and without attention-probs dropout (the mask
    rebuilt on the host by tests/_masks.py), packed against padded, bit-identical repeat calls, and guard rows past the
    packed tokens left untouched;
  * d loss / d every variable of bert_crf and bert_bilstm_crf at L = 512 against the float64 oracle, through the packed
    and padded composites and the per-kernel path;
  * short training runs of bert_cnn_crf, bert_ce and bert_mrc (pairs longer than 384 tokens) with every dropout site on;
  * bert_bilstm_crf PREDICT / EVAL at L = 512 against the oracle, the fused executor against build_graph.
"""
import ctypes
import json
import math

import numpy as np
import pytest
import torch

from _masks import attention_keep
from chinesener_b200 import _lib, autodiff, engine, fastpath, ops, synthetic, variables
from oracle import crf, crf_torch, models as omodels, nn as onn

pytestmark = pytest.mark.gpu

D = 64
SEED = (91 << 32) | 2024
CFG = {'vocab_size': 1500, 'hidden_size': 768, 'num_hidden_layers': 2, 'num_attention_heads': 12,
       'intermediate_size': 3072, 'max_position_embeddings': 512, 'type_vocab_size': 2, 'initializer_range': 0.02}

# (B, L, NH, lengths): full-length rows unless lengths are given
ATTN_CASES = [(2, 385, 2, None), (3, 448, 4, None), (1, 512, 12, None), (4, 512, 3, [512, 1, 129, 385])]


# --------------------------------------------------------------------------- attention backward kernel
def _attn_case(B, L, NH, lens):
    g = torch.Generator().manual_seed(B * L + NH)
    qkv = (torch.randn(B * L, 3 * NH * D, generator=g) * 0.7).to(torch.bfloat16)
    dctx = torch.randn(B * L, NH * D, generator=g).to(torch.bfloat16)
    lens = torch.tensor(lens if lens is not None else [L] * B)
    mask = (torch.arange(L)[None, :] < lens[:, None]).to(torch.int32)
    return qkv, dctx, mask, lens


def _attn_ref(qkv, dctx, mask, NH, keep):
    """d(sum(ctx * dctx)) / d qkv in float64, ctx = (softmax(QK^T/8 + mask term) o z) V."""
    B, L = mask.shape
    x = qkv.double().requires_grad_(True)
    q, k, v = x.view(B, L, 3, NH, D).permute(2, 0, 3, 1, 4)
    s = q @ k.transpose(-1, -2) / math.sqrt(D) + (1.0 - mask.double())[:, None, None, :] * -10000.0
    p = torch.softmax(s, -1)
    if keep < 1.0:
        p = p * (torch.from_numpy(attention_keep(B, NH, L, keep, SEED)).double() / keep)
    ctx = (p @ v).permute(0, 2, 1, 3).reshape(B * L, NH * D)
    (ctx * dctx.double()).sum().backward()
    return x.grad


def _check(got, ref):
    err = (got.float().cpu().double() - ref).abs().max().item()
    assert err < 3e-2 * ref.abs().max().item() + 1e-3, (err, ref.abs().max().item())


@pytest.mark.parametrize("keep", [1.0, 0.9])
@pytest.mark.parametrize("B,L,NH,lens", ATTN_CASES)
def test_tiled_attention_backward_padded(B, L, NH, lens, keep):
    """Padded layout: [PAD] queries carry gradients as in the kernel for L <= 384."""
    qkv, dctx, mask, _ = _attn_case(B, L, NH, lens)
    ref = _attn_ref(qkv, dctx, mask, NH, keep)
    q, m, dc = qkv.cuda(), mask.cuda(), dctx.cuda()
    ctx = ops.bert_attention(q, m, B, L, NH, D, keep_prob=keep, seed=SEED)
    d1 = ops.bert_attention_bwd(q, m, ctx, dc, B, L, NH, D, keep_prob=keep, seed=SEED)
    _check(d1, ref)
    d2 = ops.bert_attention_bwd(q, m, ctx, dc, B, L, NH, D, keep_prob=keep, seed=SEED)
    assert torch.equal(d1.view(torch.int16), d2.view(torch.int16))          # no atomics: repeat calls are bit-identical


@pytest.mark.parametrize("keep", [1.0, 0.9])
@pytest.mark.parametrize("B,L,NH,lens", ATTN_CASES)
def test_tiled_attention_backward_packed(B, L, NH, lens, keep):
    """Packed layout against float64 on the real tokens, and against the padded kernel with dctx zero on [PAD] queries."""
    qkv, dctx, mask, lens_t = _attn_case(B, L, NH, lens)
    dctx = dctx.clone()
    real = mask.view(-1).bool()
    dctx[~real] = 0                                   # [PAD] queries carry no gradient in the packed model
    ref = _attn_ref(qkv, dctx, mask, NH, keep)[real]
    q, m, dc = qkv.cuda(), mask.cuda(), dctx.cuda()
    cu, tok_src = ops.seq_pack_plan(m)
    n = int(lens_t.sum())
    qp, dp = ops.gather_rows(q, tok_src, n), ops.gather_rows(dc, tok_src, n)
    ctxp = ops.bert_attention(qp, None, B, L, NH, D, cu_seqlens=cu, keep_prob=keep, seed=SEED)
    d1 = ops.bert_attention_bwd(qp, None, ctxp, dp, B, L, NH, D, keep_prob=keep, seed=SEED, cu_seqlens=cu)
    _check(d1, ref)
    d2 = ops.bert_attention_bwd(qp, None, ctxp, dp, B, L, NH, D, keep_prob=keep, seed=SEED, cu_seqlens=cu)
    assert torch.equal(d1.view(torch.int16), d2.view(torch.int16))
    ctx = ops.bert_attention(q, m, B, L, NH, D, keep_prob=keep, seed=SEED)
    dpad = ops.gather_rows(ops.bert_attention_bwd(q, m, ctx, dc, B, L, NH, D, keep_prob=keep, seed=SEED), tok_src, n)
    assert float((d1.float() - dpad.float()).abs().max()) <= 2e-2 * float(dpad.float().abs().max())


def test_tiled_attention_backward_leaves_guard_rows():
    """Through the C-ABI with an over-allocated d_qkv: rows past the packed tokens keep their sentinel values."""
    B, L, NH = 3, 448, 4
    qkv, dctx, mask, lens = _attn_case(B, L, NH, [448, 5, 400])
    m = mask.cuda()
    cu, tok_src = ops.seq_pack_plan(m)
    n = int(lens.sum())
    qp, dp = ops.gather_rows(qkv.cuda(), tok_src, n), ops.gather_rows(dctx.cuda(), tok_src, n)
    ctxp = ops.bert_attention(qp, None, B, L, NH, D, cu_seqlens=cu)
    ref = ops.bert_attention_bwd(qp, None, ctxp, dp, B, L, NH, D, cu_seqlens=cu)
    guard = 37
    out = torch.full((n + guard, 3 * NH * D), 1234.0, dtype=torch.bfloat16, device="cuda")
    rc = _lib.lib().ner_bert_attention_bwd_packed(_lib.ptr(qp), _lib.ptr(cu), _lib.ptr(ctxp), _lib.ptr(dp), _lib.ptr(out),
                                                  B, L, NH, D, 0.125, 1.0, 0, _lib.stream())
    assert rc == 0
    assert torch.equal(out[:n], ref)
    assert bool((out[n:] == 1234.0).all())


# --------------------------------------------------------------------------- plugins
def _batch(lens, L, vocab, seed):
    """MSRA-shaped features with the given sentence lengths (including [CLS] / [SEP])."""
    f = synthetic.msra_batch(len(lens), L, vocab=vocab, seed=seed, full=True)
    for b, n in enumerate(lens):
        f['token_ids'][b, n - 1] = 102
        f['label_ids'][b, n - 1] = 9
        for k in ('token_ids', 'label_ids', 'mask'):
            f[k][b, n:] = 0
        f['seq_len'][b] = n
    return f


def _est(tmp_path, model, lens, L, dropout=0.0, bert_dropout=0.0, **extra):
    cfg = dict(CFG, hidden_dropout_prob=bert_dropout, attention_probs_dropout_prob=bert_dropout)
    (tmp_path / "bert_config.json").write_text(json.dumps(cfg))
    feats = _batch(lens, L, CFG['vocab_size'], seed=31)
    params = dict(synthetic.data_params(L), pretrain_dir=str(tmp_path), embedding_dropout=dropout, **extra)
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


@pytest.mark.parametrize("mode", ["packed", "padded", "per_kernel"])
@pytest.mark.parametrize("model", ["bert_crf", "bert_bilstm_crf"])
def test_gradients_at_512_match_oracle_autograd(tmp_path, model, mode, monkeypatch):
    from chinesener_b200 import bert as _bert
    from chinesener_b200.tools import layer as _layer
    monkeypatch.setattr(_layer, "TRAIN_PACK", mode == "packed")
    monkeypatch.setattr(_bert, "PER_KERNEL", mode == "per_kernel")
    # tanh cells: the plugin's default ReLU cell is unbounded, and over a 512-step recurrence it amplifies the bf16
    # rounding of the encoder output.  On an H100 its embedding gradients are 18% of scale from float64 at L = 512 and
    # 6.6% already at L = 256 (the whole-head attention kernel), in every encoder mode; with tanh cells they are 0.4%.
    est, feats = _est(tmp_path, model, [512, 37], 512, keep_prob_list=[1.0], rnn_activation='tanh')
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
        scale = max(g_ref.abs().max().item(), 1e-3 * gscale)   # key biases have an analytically zero gradient
        worst[name] = (g - g_ref).abs().max().item() / scale
    bad = {k: v for k, v in worst.items() if v > 8e-2}
    print(model, mode, "max relative gradient error:", max(worst.values()), "over", len(worst), "variables")
    assert not bad, bad


def _mrc_query_ids():
    rng = np.random.default_rng(7)
    return {n: rng.integers(106, CFG['vocab_size'], size=k).tolist() for n, k in {'ORG': 22, 'PER': 10, 'LOC': 20}.items()}


@pytest.mark.parametrize("model,L,lens,lr", [("bert_cnn_crf", 512, [512, 60, 23], 2e-5),
                                             ("bert_ce", 512, [512, 60, 23], 5e-5),
                                             ("bert_mrc", 384, [384, 60, 23], 5e-5)])
def test_training_runs_at_long_lengths(tmp_path, model, L, lens, lr):
    extra = dict(cnn_dropout=0.1) if model == "bert_cnn_crf" else {}
    if model == "bert_mrc":
        extra['mrc_query_ids'] = _mrc_query_ids()            # pairs of up to 22 + 2 + 384 = 408 tokens
    est, feats = _est(tmp_path, model, lens, L, dropout=0.1, bert_dropout=0.1, **extra)
    if model == "bert_mrc":
        from chinesener_b200.data import mrc
        assert mrc.device_table(est.params).L2 > 384
    est.params.update(lr=lr, num_train_steps=100, warmup_ratio=0.1)
    losses = [float(est.train_step(feats)) for _ in range(12)]
    print(model, "losses:", ["%.3f" % v for v in losses])
    assert np.isfinite(losses).all(), losses
    assert losses[-1] < 0.8 * losses[0], losses


def test_bert_bilstm_crf_predict_and_eval_at_512(tmp_path):
    """Same bars as tests/test_models_gpu.py::test_bert_models_match_oracle, plus the fused executor."""
    from chinesener_b200.tools import layer
    L = 512
    est, feats = _est(tmp_path, "bert_bilstm_crf", [512, 300, 77, 9], L)
    est.evaluate(feats)
    est.store.vars["logits/kernel"].mul_(8.0)
    est.store.touch()
    out = est.evaluate(feats)
    dev = est.to_device(feats)
    fused = fastpath.bert_bilstm_crf_predict(est, dev)
    assert fused is not None
    _, ref_pred = est.forward_device(dev, False)
    assert torch.equal(fused, ref_pred)
    pred = ref_pred.cpu().numpy()
    np.testing.assert_array_equal(out['pred_ids'].numpy(), pred)
    w = est.store.state_dict()
    p = dict(est.params, num_hidden_layers=2, num_attention_heads=12)
    ref_emul = omodels.bert_bilstm_crf(w, feats, p, dtype=torch.float64, emulate_bf16=True)
    ref_true = omodels.bert_bilstm_crf(w, feats, p, dtype=torch.float64, emulate_bf16=False)
    with variables.use_store(est.store):
        emb = layer.pretrain_bert_embedding(dev['token_ids'], dev['mask'], dev['segment_ids'], est.params['pretrain_dir'], 0.1,
                                            False)
        x = layer.bilstm(emb, 'lstm', est.params['rnn_activation'], [128], [1.0], 1, dev['seq_len'], 'float32', False)
        logits = layer.dense(x, 10, 'logits')
    lg = logits.cpu().double()
    valid = torch.arange(L)[None, :] < feats['seq_len'][:, None]
    err_emul = (lg - ref_emul['logits'])[valid].abs().max().item()
    err_true = (lg - ref_true['logits'])[valid].abs().max().item()
    print(f"L=512: max|logit - oracle(bf16-emulated)| = {err_emul:.2e}, vs fp64 oracle = {err_true:.2e}")
    assert err_emul < 4e-3 * max(1.0, ref_emul['logits'][valid].abs().max().item())
    assert err_true < 5e-2 * max(1.0, ref_true['logits'][valid].abs().max().item() / 8.0)
    trans = w['crf_layer/transitions'].numpy()
    own, _ = crf.crf_decode(logits.cpu().numpy(), trans, feats['seq_len'].numpy(), dtype=np.float32)
    np.testing.assert_array_equal(pred, own)
    ll_ref = crf.crf_log_likelihood(logits.cpu().numpy(), feats['label_ids'].numpy(), feats['seq_len'].numpy(), trans)
    assert abs(out['loss'] - float(np.mean(-ll_ref))) < 1e-3 * max(1.0, abs(out['loss']))
    agree = (pred == ref_emul['pred_ids']).mean()
    assert agree > 0.99, agree
