# -*-coding:utf-8 -*-
"""GPU: the bert_mrc_span plugin (span-pointer MRC NER) and its kernels ner_mrc_span_targets / _match_fwd / _match_bwd /
_decode, against the float64 restatement of tests/_mrc_span_oracle.py.

  * targets bit-exact for T in {1, 3, 32} and seq_len in {0, 1, 2, 3, L}, guard words untouched;
  * match forward: z within 2e-3 of max |z| and the loss within 1e-4 relative, at keep 1.0 and 0.9, three shapes;
  * match backward: dU | dV, db1, dw2, db2 within 1e-2 of scale against float64 autograd, repeat calls bit-identical;
  * decode: spans, counts and pred_ids bit-exact against the restatement fed the forward kernel's z (the decode evaluates
    the same tile arithmetic), probabilities within 1 ulp; crafted nesting, two ends for one start, count > cap;
  * plugin: PREDICT / EVAL against the restatement (bf16 and fp32 encoders), gradients of every variable (packed and
    padded training encoders), a 12-step AdamW run, no device sync in PREDICT, the driver pickle and InferHelper.
"""
import ctypes
import json
import os
import pickle

import numpy as np
import pytest
import torch

import _mrc_span_oracle as so
from _mrc_oracle import mrc_pairs as oracle_pairs
from chinesener_b200 import _lib, autodiff, engine, evaluation, ops, synthetic, variables
from chinesener_b200.data import mrc
from oracle import nn as onn

pytestmark = pytest.mark.gpu

SMALL_BERT = {'vocab_size': 3000, 'hidden_size': 768, 'num_hidden_layers': 2, 'num_attention_heads': 12,
              'intermediate_size': 3072, 'max_position_embeddings': 512, 'type_vocab_size': 2, 'initializer_range': 0.02}
QUERY_LENS = {'ORG': 22, 'PER': 10, 'LOC': 20}


def _query_ids(seed=7, vocab=3000):
    rng = np.random.default_rng(seed)
    return {n: rng.integers(106, vocab, size=k).tolist() for n, k in QUERY_LENS.items()}


def _lens(P, L, seed):
    lens = np.random.default_rng(seed).integers(0, L + 1, size=P).astype(np.int32)
    for q, v in enumerate([L, 0, 1, 2, 3]):
        if q < P:
            lens[q] = v
    return lens


# --------------------------------------------------------------------------- targets
@pytest.mark.parametrize("T", [1, 3, 32])
def test_targets_bit_exact_with_guards(T):
    P, L = 5 * T, 40
    rng = np.random.default_rng(T)
    labels = rng.choice([0, 0, 1, 2, 2], size=(P, L)).astype(np.int32)
    lens = _lens(P, L, seed=T)
    ref = so.targets(labels, lens)
    guard, sentinel = 29, -5
    outs = [torch.full((P * L + guard,), sentinel, dtype=torch.int32, device='cuda') for _ in range(3)]
    lab, sl = torch.from_numpy(labels).cuda(), torch.from_numpy(lens).cuda()
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    assert _lib.lib().ner_mrc_span_targets(p(lab), p(sl), P, L, p(outs[0]), p(outs[1]), p(outs[2]), None) == 0
    torch.cuda.synchronize()
    for got, want in zip(outs, ref):
        got = got.cpu().numpy()
        np.testing.assert_array_equal(got[:P * L], want.reshape(-1))
        assert (got[P * L:] == sentinel).all()
    for got, want in zip(ops.mrc_span_targets(lab, sl), ref):
        np.testing.assert_array_equal(got.cpu().numpy(), want)


# --------------------------------------------------------------------------- match head
def _head_case(P, L, I, seed, scale=1.0):
    g = torch.Generator(device='cuda').manual_seed(seed)
    U = torch.randn(P, L, I, generator=g, device='cuda') * scale
    V = torch.randn(P, L, I, generator=g, device='cuda') * scale
    b1 = 0.3 * torch.randn(I, generator=g, device='cuda')
    w2 = torch.randn(I, generator=g, device='cuda') / I ** 0.5
    b2 = torch.tensor([0.05], device='cuda')
    lens = _lens(P, L, seed)
    labels = np.random.default_rng(seed).choice([0, 0, 0, 1, 2, 2], size=(P, L)).astype(np.int32)
    span_end = so.targets(labels, lens)[2]
    uv = torch.cat([U, V], -1).reshape(P * L, 2 * I).contiguous()
    return uv, U, V, b1, w2, b2, lens, span_end


def _ref_forward(U, V, b1, w2, b2, lens, span_end, keep, seed):
    d = lambda t: t.double()
    z = so.match_logits(d(U), d(V), d(b1), d(w2), d(b2)[0], lens, keep=keep, seed=seed)
    return z, so.bce_loss(z, span_end, lens)


@pytest.mark.parametrize("keep", [1.0, 0.9])
@pytest.mark.parametrize("P,L,I", [(3, 7, 64), (192, 128, 1024), (6, 480, 1024)])
def test_match_forward_against_float64(P, L, I, keep):
    seed = 0x1234_5678_9ABC
    uv, U, V, b1, w2, b2, lens, span_end = _head_case(P, L, I, seed=P + L)
    sl, se = torch.from_numpy(lens).cuda(), torch.from_numpy(span_end).cuda()
    z, loss = ops.mrc_span_match_fwd(uv, b1, w2, b2, sl, L, se, keep, seed)
    z_ref, loss_ref = _ref_forward(U, V, b1, w2, b2, lens, span_end, keep, seed)
    cand = torch.from_numpy(so.candidates(lens, L)).cuda()
    scale = z_ref[cand].abs().max().item()
    err = (z.double() - z_ref)[cand].abs().max().item()
    print(f"match fwd P={P} L={L} I={I} keep={keep}: max|z - ref| = {err:.2e} (max|z| {scale:.2f}), "
          f"loss {float(loss):.6f} vs {float(loss_ref):.6f}")
    assert err <= 2e-3 * scale
    assert (z[~cand] == 0).all()
    assert abs(float(loss) - float(loss_ref)) <= 1e-4 * abs(float(loss_ref))
    z2, loss2 = ops.mrc_span_match_fwd(uv, b1, w2, b2, sl, L, se, keep, seed)
    assert torch.equal(z, z2) and torch.equal(loss, loss2)
    # padded rows: a wider uv buffer (row stride > 2I) gives the same z
    wide = torch.zeros((P * L, 2 * I + 32), device='cuda')
    wide[:, :2 * I] = uv
    assert torch.equal(ops.mrc_span_match_fwd(wide, b1, w2, b2, sl, L, se, keep, seed)[0], z)


@pytest.mark.parametrize("P,L,I,keep", [(3, 7, 64, 1.0), (24, 64, 256, 0.9), (192, 128, 1024, 1.0)])
def test_match_backward_against_float64_autograd(P, L, I, keep):
    seed = 987654321
    uv, U, V, b1, w2, b2, lens, span_end = _head_case(P, L, I, seed=P + I)
    sl, se = torch.from_numpy(lens).cuda(), torch.from_numpy(span_end).cuda()
    z, loss = ops.mrc_span_match_fwd(uv, b1, w2, b2, sl, L, se, keep, seed)
    got = ops.mrc_span_match_bwd(uv, z, b1, w2, sl, se, 0.75, keep, seed)
    again = ops.mrc_span_match_bwd(uv, z, b1, w2, sl, se, 0.75, keep, seed)
    assert all(torch.equal(a, b) for a, b in zip(got, again))
    leaves = [t.double().clone().requires_grad_(True) for t in (U, V, b1, w2, b2)]
    z_ref = so.match_logits(*leaves[:4], leaves[4][0], lens, keep=keep, seed=seed)
    (0.75 * so.bce_loss(z_ref, span_end, lens)).backward()
    d_uv = got[0].view(P, L, 2 * I)
    pairs = [("dU", d_uv[..., :I], leaves[0].grad), ("dV", d_uv[..., I:], leaves[1].grad), ("db1", got[1], leaves[2].grad),
             ("dw2", got[2], leaves[3].grad), ("db2", got[3], leaves[4].grad)]
    for name, g, ref in pairs:
        rel = ((g.double() - ref).norm() / ref.norm().clamp_min(1e-30)).item()
        print(f"match bwd P={P} L={L} I={I} keep={keep}: {name} norm-relative error {rel:.2e}")
        assert rel <= 1e-2, name


# --------------------------------------------------------------------------- decode
def _decode_case(B, T, L, I, seed, density=0.5):
    rng = np.random.default_rng(seed)
    P = B * T
    uv, U, V, b1, w2, b2, _, _ = _head_case(P, L, I, seed=seed, scale=0.5)
    lens = _lens(B, L, seed)
    sl = (rng.normal(size=(P, L, 2)) + np.array([0.0, 2 * density - 1.0])).astype(np.float32)
    el = (rng.normal(size=(P, L, 2)) + np.array([0.0, 2 * density - 1.0])).astype(np.float32)
    tt = [[2 + 2 * t, 3 + 2 * t] for t in range(T)]
    return uv, b1, w2, b2, lens, sl, el, tt


def _kernel_z(uv, b1, w2, b2, lens, T, L):
    pair_lens = torch.from_numpy(np.repeat(lens, T)).cuda()
    return ops.mrc_span_match_fwd(uv, b1, w2, b2, pair_lens, L)[0].cpu().numpy()


def _check_decode(uv, b1, w2, b2, lens, sl, el, tt, cap=None):
    T, (P, L, _) = len(tt), sl.shape
    cap = L if cap is None else cap
    pred = ops.mrc_span_decode(torch.from_numpy(sl).cuda(), torch.from_numpy(el).cuda(), uv, b1, w2, b2,
                               torch.from_numpy(lens).cuda(), torch.tensor(tt, dtype=torch.int32, device='cuda'), 1, 8, 9,
                               cap=cap)
    z = _kernel_z(uv, b1, w2, b2, lens, T, L)
    ref_pred, words, probs, counts = so.decode(sl, el, z, lens, tt, 1, 8, 9, cap)
    got_counts = pred.span_counts.cpu().numpy()
    np.testing.assert_array_equal(got_counts, counts)
    np.testing.assert_array_equal(pred.cpu().numpy(), ref_pred)
    gw, gp = pred.spans.cpu().numpy(), pred.span_probs.cpu().numpy()
    for b in range(len(lens)):
        n = min(int(counts[b]), cap)
        np.testing.assert_array_equal(gw[b, :n], words[b, :n])
        np.testing.assert_allclose(gp[b, :n], probs[b, :n], rtol=2.4e-7, atol=0)
    return pred, counts


@pytest.mark.parametrize("B,T,L,I", [(8, 3, 40, 64), (4, 32, 24, 32), (16, 3, 128, 1024)])
def test_decode_matches_restatement(B, T, L, I):
    case = _decode_case(B, T, L, I, seed=B * T + L)
    pred, counts = _check_decode(*case)
    assert counts.sum() > 0
    # repeat calls are bit-identical
    pred2, _ = _check_decode(*case)
    assert torch.equal(pred, pred2) and torch.equal(pred.spans, pred2.spans)


def test_decode_crafted_nesting_two_ends_and_cap():
    L, I, T = 10, 32, 2
    uv = torch.randn(T * L, 2 * I, device='cuda')
    b1, w2 = torch.zeros(I, device='cuda'), torch.zeros(I, device='cuda')
    b2 = torch.tensor([1.0], device='cuda')                     # every start x end pair scores z = 1
    sl = np.zeros((T, L, 2), np.float32)
    el = np.zeros((T, L, 2), np.float32)
    sl[0, 1, 1] = el[0, 2, 1] = el[0, 4, 1] = 1.0               # type 0: one start, two ends
    sl[1, 2, 1] = el[1, 3, 1] = 1.0                             # type 1: nested inside type 0's 1..4
    tt = [[2, 3], [4, 5]]
    pred, counts = _check_decode(uv, b1, w2, b2, np.array([9], np.int32), sl, el, tt, cap=2)
    assert counts.tolist() == [3]                               # one more than cap: counted, not stored
    assert pred.spans.cpu().tolist() == [[1 | 3 << 12, 1 | 5 << 12]]
    assert pred.cpu().tolist() == [[8, 2, 3, 1, 1, 1, 1, 1, 9, 0]]   # ties: type 0, then the lower end
    full = ops.mrc_span_decode(torch.from_numpy(sl).cuda(), torch.from_numpy(el).cuda(), uv, b1, w2, b2,
                               torch.tensor([9], dtype=torch.int32, device='cuda'),
                               torch.tensor(tt, dtype=torch.int32, device='cuda'), 1, 8, 9)
    assert full.spans[0, :3].cpu().tolist() == [1 | 3 << 12, 1 | 5 << 12, 2 | 4 << 12 | 1 << 24]


# --------------------------------------------------------------------------- plugin
def _estimator(tmp_path, B, L, seed, **extra):
    (tmp_path / "bert_config.json").write_text(json.dumps(SMALL_BERT))
    feats = synthetic.msra_batch(B, L, vocab=SMALL_BERT['vocab_size'], seed=seed)
    est = engine.Estimator("bert_mrc_span", dict(synthetic.data_params(L), pretrain_dir=str(tmp_path),
                                                 mrc_query_ids=_query_ids(), **extra))
    est.evaluate(feats)                                         # creates the variables
    for n in ("start_logits/kernel", "end_logits/kernel"):
        est.store.vars[n].mul_(8.0)                             # decisive start / end decisions
    est.store.vars["span_logits/classifier2/kernel"].mul_(4.0)
    est.store.touch()
    return est, feats


def _cuda_heads(est, dev):
    """The plugin's start / end logits [B*T, L, 2] and U | V rows, by the same calls as build_graph."""
    from chinesener_b200.model import _blocks, bert_mrc, bert_mrc_span
    from chinesener_b200.tools import layer
    table = mrc.device_table(est.params)
    B, L = dev['token_ids'].shape
    with est._layer_settings(dev), variables.use_store(est.store):
        pr = ops.mrc_pairs(dev['token_ids'], dev['seq_len'], table.query_ids, table.query_len, table.type_tag, table.L2,
                           table.sep_id)
        pr['mask'].total_tokens = table.pair_tokens(dev['mask'])
        hidden = _blocks.bert_sequence({'token_ids': pr['ids'], 'mask': pr['mask'], 'segment_ids': pr['segment_ids']},
                                       est.params, False)
        rows = bert_mrc.sentence_rows(hidden, pr['align'], B * table.T, L, False)
        w1 = est.store.vars["span_logits/classifier1/kernel"]
        return layer.dense(rows, 2, 'start_logits'), layer.dense(rows, 2, 'end_logits'), \
            bert_mrc_span.span_projection(rows, w1, False)


def span_oracle(w, features, table, emulate_bf16, num_layers=2):
    """pairs -> BertModel -> alignment -> start / end dense + CE, U | V (bf16 operands) -> match head + BCE (float64)."""
    B, L = features['token_ids'].shape
    pr = oracle_pairs(features['token_ids'].numpy(), features['seq_len'].numpy(), table.query_ids.cpu().numpy(),
                      table.query_len.cpu().numpy(), table.type_tag.cpu().numpy(), table.L2, table.sep_id,
                      features['label_ids'].numpy())
    t = lambda a: torch.from_numpy(a)
    seq = onn.bert_encoder(w, t(pr['ids']), t(pr['mask']), t(pr['segment_ids']), num_layers=num_layers, num_heads=12,
                           dtype=torch.float64, emulate_bf16=emulate_bf16)
    H = seq.shape[-1]
    P = B * table.T
    rows = seq.reshape(-1, H)[t(pr['align']).long()].view(P, L, H)
    r = onn._rb(rows, emulate_bf16)
    start = onn.dense(r, w["start_logits/kernel"].double(), w["start_logits/bias"].double())
    end = onn.dense(r, w["end_logits/kernel"].double(), w["end_logits/bias"].double())
    w1 = w["span_logits/classifier1/kernel"].double()
    r16, w16 = onn._rb(rows, True), onn._rb(w1, True)           # the projection GEMM takes bf16 operands
    U, V = r16 @ w16[:H], r16 @ w16[H:]
    z = so.match_logits(U, V, w["span_logits/classifier1/bias"].double(), w["span_logits/classifier2/kernel"].double()[:, 0],
                        w["span_logits/classifier2/bias"].double()[0], pr['seq_len'])
    st, en, span_end = so.targets(pr['labels'], pr['seq_len'])
    xent = lambda lg, y: _masked_xent(lg, t(y), t(pr['seq_len']))
    loss = xent(start, st) + xent(end, en) + so.bce_loss(z, span_end, pr['seq_len'])
    return dict(start=start, end=end, z=z, loss=loss, pairs=pr)


def _masked_xent(logits, labels, seq_len):
    B, L, _ = logits.shape
    valid = torch.arange(L)[None, :] < seq_len.long()[:, None]
    ce = torch.logsumexp(logits, -1) - logits.gather(-1, labels.long()[..., None])[..., 0]
    n = int(valid.sum())
    return (ce * valid).sum() / n if n > 0 else (ce * 0.0).sum()


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_predict_and_eval_match_restatement(tmp_path, precision):
    B, L = 6, 48
    est, feats = _estimator(tmp_path, B, L, seed=5, bert_precision=precision, mrc_span_hidden=256)
    table = mrc.device_table(est.params)
    out = est.evaluate(feats)
    res = est.predict(feats)
    pred = res['pred_ids'].numpy()
    np.testing.assert_array_equal(out['pred_ids'].numpy(), pred)
    dev = est.to_device(feats)
    sl, el, uv = _cuda_heads(est, dev)
    T = table.T
    w = est.store.state_dict()
    b1, w2, b2 = (w[f"span_logits/{n}"] for n in ("classifier1/bias", "classifier2/kernel", "classifier2/bias"))
    z = _kernel_z(uv, b1.cuda(), w2.cuda().view(-1), b2.cuda(), feats['seq_len'].numpy(), T, L)
    ref_pred, words, probs, counts = so.decode(sl.cpu().numpy(), el.cpu().numpy(), z, feats['seq_len'].numpy(),
                                               table.type_tag.tolist(), table.o_tag, table.cls_tag, table.sep_tag, L)
    np.testing.assert_array_equal(pred, ref_pred)               # the decode of the plugin's own heads, bit for bit
    assert counts.sum() > 0 and ((pred >= 2) & (pred <= 7)).any()
    assert (counts > L).any()                                   # random weights: more spans than the default cap
    for b, spans in enumerate(res['pred_spans']):
        assert len(spans) == min(counts[b], L)
        for (name, s, e, p), wd, pr in zip(spans, words[b], probs[b]):
            assert (s, e, table.names.index(name)) == (int(wd) & 0xFFF, (int(wd) >> 12) & 0xFFF, int(wd) >> 24)
            assert abs(p - float(pr)) <= 2.4e-7 * pr
    ref = span_oracle(w, feats, table, emulate_bf16=precision == 'bf16')
    pair_len = torch.from_numpy(ref['pairs']['seq_len'])
    valid = torch.arange(L)[None, :] < pair_len[:, None]
    for name, got, want in (("start", sl, ref['start']), ("end", el, ref['end'])):
        scale = want[valid].abs().max().item()
        err = (got.cpu().double() - want)[valid].abs().max().item()
        print(f"bert_mrc_span {precision}: max|{name} logit - restatement| = {err:.2e} (scale {scale:.2f})")
        assert err < 2e-2 * scale
    cand = torch.from_numpy(so.candidates(ref['pairs']['seq_len'], L))
    zscale = ref['z'][cand].abs().max().item()
    zerr = (torch.from_numpy(z).double() - ref['z'])[cand].abs().max().item()
    print(f"bert_mrc_span {precision}: max|z - restatement| = {zerr:.2e} (scale {zscale:.2f}); loss {out['loss']:.5f} vs "
          f"{float(ref['loss']):.5f}")
    assert zerr < 2e-2 * zscale
    assert abs(out['loss'] - float(ref['loss'])) < 1e-2 * abs(float(ref['loss']))
    assert torch.equal(est.predict(feats)['pred_ids'], torch.from_numpy(pred))
    assert est.evaluate(feats)['loss'] == out['loss']


def test_predict_has_no_device_sync(tmp_path):
    est, feats = _estimator(tmp_path, 16, 64, seed=9)
    dev = est.to_device(feats)
    ref = est.predict_device(dev)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        pred = est.predict_device(dev)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.equal(pred, ref) and torch.equal(pred.spans, ref.spans)


CFG_TRAIN = {'vocab_size': 1500, 'hidden_size': 768, 'num_hidden_layers': 2, 'num_attention_heads': 12,
             'intermediate_size': 3072, 'max_position_embeddings': 128, 'type_vocab_size': 2, 'initializer_range': 0.02}


def _train_est(tmp_path, dropout=0.0, bert_dropout=0.0, span_dropout=0.0, B=4, L=32):
    cfg = dict(CFG_TRAIN, hidden_dropout_prob=bert_dropout, attention_probs_dropout_prob=bert_dropout)
    (tmp_path / "bert_config.json").write_text(json.dumps(cfg))
    feats = synthetic.msra_batch(B, L, vocab=CFG_TRAIN['vocab_size'], seed=21)
    feats['seq_len'][1] = 0                                     # an empty sentence: empty pairs
    feats['mask'][1] = 0
    feats['token_ids'][1] = 0
    feats['label_ids'][1] = 0
    params = dict(synthetic.data_params(L), pretrain_dir=str(tmp_path), embedding_dropout=dropout, mrc_span_hidden=64,
                  mrc_dropout=span_dropout, mrc_query_ids=_query_ids(vocab=CFG_TRAIN['vocab_size']))
    return engine.Estimator("bert_mrc_span", params), feats


@pytest.mark.parametrize("packed", [True, False])
def test_gradients_match_restatement_autograd(tmp_path, packed, monkeypatch):
    from chinesener_b200.tools import layer as _layer
    monkeypatch.setattr(_layer, "TRAIN_PACK", packed)
    est, feats = _train_est(tmp_path)
    est.evaluate(feats)
    for n in ("start_logits/kernel", "end_logits/kernel"):
        est.store.vars[n].mul_(4.0)
    est.store.touch()
    table = mrc.device_table(est.params)
    w = est.store.state_dict()
    wd = {k: v.double().clone().requires_grad_(True) for k, v in w.items()}
    ref = span_oracle(wd, feats, table, emulate_bf16=False)
    ref['loss'].backward()
    dev = est.to_device(feats)
    with variables.use_store(est.store), autodiff.recording(est.store) as tape:
        loss, pred = est.build_graph(dev, None, est.params, True)
        tape.backward()
    ref_loss = float(ref['loss'].detach())
    assert abs(float(loss) - ref_loss) < 2e-2 * max(1.0, abs(ref_loss))
    assert pred.shape == feats['label_ids'].shape and pred.dtype == torch.int32
    grads = {k: v.grad for k, v in wd.items()}
    gscale = max(g.abs().max().item() for n, g in grads.items() if g is not None and "pooler" not in n)
    worst = {}
    for name, g_ref in grads.items():
        if g_ref is None or "pooler" in name:
            continue
        g = est.store.grads[name].cpu().double()
        scale = max(g_ref.abs().max().item(), 1e-3 * gscale)
        worst[name] = (g - g_ref).abs().max().item() / scale
    assert all(f"span_logits/{n}" in worst for n in ("classifier1/kernel", "classifier1/bias", "classifier2/kernel",
                                                     "classifier2/bias"))
    bad = {k: v for k, v in worst.items() if v > 8e-2}
    print("max relative gradient error:", max(worst.values()), "over", len(worst), "variables")
    assert not bad, bad


def test_training_reduces_loss(tmp_path):
    est, feats = _train_est(tmp_path, dropout=0.1, bert_dropout=0.1, span_dropout=0.1)
    est.params.update(lr=5e-5, num_train_steps=100, warmup_ratio=0.1)
    losses = [float(est.train_step(feats)) for _ in range(12)]
    print("bert_mrc_span losses:", ["%.3f" % v for v in losses])
    assert np.isfinite(losses).all(), losses
    assert losses[-1] < 0.8 * losses[0], losses


def test_driver_writes_prediction_pickle(tmp_path):
    from chinesener_b200 import main as driver
    from test_main_driver_gpu import L as DRIVER_L, _setup
    root, pre = _setup(tmp_path)
    vocab = ['[PAD]', '[UNK]', '[CLS]', '[SEP]'] + sorted(set(''.join(mrc.DEFAULT_QUERIES.values())))
    with open(os.path.join(pre, 'vocab.txt'), 'w', encoding='utf-8') as f:
        f.write('\n'.join(vocab) + '\n')
    cfg_path = os.path.join(pre, 'bert_config.json')
    cfg = json.load(open(cfg_path))
    cfg['vocab_size'] = max(cfg['vocab_size'], len(vocab))
    json.dump(cfg, open(cfg_path, 'w'))
    with pytest.warns(UserWarning):
        s = driver.main(['--model_name', 'bert_mrc_span', '--data', 'msra', '--data_dir', os.path.join(root, 'msra'),
                         '--checkpoint_root', str(tmp_path / 'ckpt'), '--pretrain_dir', pre, '--epoch_size', '2',
                         '--batch_size', '4'])
    assert s['n_predict'] == 24
    path = os.path.join(root, 'msra', 'bert_mrc_span_predict.pkl')
    pred = pickle.load(open(path, 'rb'))
    assert len(pred) == 24
    assert all(p['pred_ids'].shape == (DRIVER_L,) and p['pred_ids'].dtype == np.int32 for p in pred)
    assert np.isfinite(s['entity_micro_f1'])
    from chinesener_b200.data.records import NerDataset
    idx2tag = NerDataset(os.path.join(root, 'msra'), 4, 2, 'bert_mrc_span').params['idx2tag']
    tag_rep, ent_rep = evaluation.SingleEval(path, idx2tag).gen_report()
    assert 0.0 <= ent_rep['micro avg']['f1-score'] <= 1.0


def test_infer_helper_returns_the_spans(tmp_path):
    from chinesener_b200.data.tokenizer import FullTokenizer
    from chinesener_b200.inference import InferHelper, TAG2IDX
    from chinesener_b200.tools.infer_utils import span_entities
    gold = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "warmup_features.json"), encoding="utf8"))
    vocab = dict(gold["bert_vocab_subset"])
    vocab.setdefault("[UNK]", 100)
    (tmp_path / "bert_config.json").write_text(json.dumps(dict(SMALL_BERT, vocab_size=21128)))
    params = dict(synthetic.data_params(150), pretrain_dir=str(tmp_path), mrc_query_ids=_query_ids(vocab=21128))
    est = engine.Estimator("bert_mrc_span", params)
    helper = InferHelper(150, TAG2IDX, "bert_mrc_span", FullTokenizer(vocab), estimator=est)
    text = gold["text"]
    helper.infer(text)                                           # first call creates the variables
    for n in ("start_logits/kernel", "end_logits/kernel"):
        est.store.vars[n].mul_(8.0)
    est.store.touch()
    texts = [text, text[:7], text[3:30], text[::2]]
    batch = [dict(e) for e in helper.infer_batch(texts)]
    feats = [dict(helper.make_feature(t)) for t in texts]
    from chinesener_b200.data.base_preprocess import features_to_batch
    res = est.predict(features_to_batch(feats))
    joined = [dict(e) for e in span_entities([f['tokens'] for f in feats], res['pred_spans'])]
    assert batch == joined
    assert any(batch)
    # infer() on one sentence: the host join of that batch's spans (a different row count may tile the encoder GEMMs
    # differently, so it is compared with its own batch, not with infer_batch)
    one = est.predict(features_to_batch([dict(helper.make_feature(text))]))
    assert dict(helper.infer(text)) == dict(span_entities([helper.make_feature(text)['tokens']], one['pred_spans'])[0])
