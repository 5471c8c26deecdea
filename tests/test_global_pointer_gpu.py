# -*-coding:utf-8 -*-
"""GPU: the bert_global_pointer plugin and its kernels ner_gp_targets / _rope / _rope_bwd / _loss_fwd / _loss_bwd / _decode,
against the float64 restatement of tests/_gp_oracle.py.

  * targets bit-exact (ill-formed BIO, seq_len in {0, 1, 2, 3, L});
  * RoPE: hi + lo of the split mode within 1e-6 of scale (plus the 2^-16 of the bf16 pair) of float64, its backward within
    1e-6 of scale;
  * loss: within 1e-4 relative of float64 on the same bf16 operands, split mode within 1e-5 on its own hi + lo operands;
  * backward: dQ' / dK' within 1e-2 of scale against float64 autograd;
  * decode: spans, counts and pred_ids bit-exact against the restatement fed the kernel's own s; split-mode signs against
    float64 where |s| > 1e-4; crafted nesting and count > cap;
  * packed and padded rows bit-identical, repeat calls bit-identical;
  * plugin: PREDICT / EVAL against the restatement (bf16 and fp32 encoders), gradients of every variable (packed and
    padded training encoders), an AdamW run, no device sync in PREDICT, the driver pickle, 'pred_spans' and InferHelper.
"""
import json
import os
import pickle

import numpy as np
import pytest
import torch

import _gp_oracle as gp
from chinesener_b200 import autodiff, engine, evaluation, ops, synthetic, variables
from chinesener_b200.data import mrc
from oracle import nn as onn

pytestmark = pytest.mark.gpu

D = gp.D
SMALL_BERT = {'vocab_size': 3000, 'hidden_size': 768, 'num_hidden_layers': 2, 'num_attention_heads': 12,
              'intermediate_size': 3072, 'max_position_embeddings': 512, 'type_vocab_size': 2, 'initializer_range': 0.02}
TYPE_TAG = lambda T: [[2 + 2 * t, 3 + 2 * t] for t in range(T)]


def _lens(B, L, seed):
    lens = np.random.default_rng(seed).integers(0, L + 1, size=B).astype(np.int32)
    for q, v in enumerate([L, 0, 1, 2, 3]):
        if q < B and B > 5:
            lens[q] = v
    if B <= 5:
        lens[0] = L
    return lens


def _labels(B, L, T, seed):
    """Tag ids 0 [PAD], 1 O, 2 + 2t B-X_t, 3 + 2t I-X_t, drawn so that runs, ill-formed I-runs and single B's occur."""
    rng = np.random.default_rng(seed)
    return rng.choice([1, 1, 1] + list(range(2, 2 + 2 * T)) + [3] * 2, size=(B, L)).astype(np.int32)


def _case(B, T, L, seed, scale=1.0):
    g = torch.Generator(device='cuda').manual_seed(seed)
    proj = torch.randn(B * L, T * 2 * D, generator=g, device='cuda') * scale
    lens = _lens(B, L, seed)
    labels = _labels(B, L, T, seed)
    return proj, lens, labels


def _t(a, dtype=None):
    return torch.as_tensor(a, device='cuda') if dtype is None else torch.as_tensor(a, dtype=dtype, device='cuda')


def _rot64(proj, B, L, T):
    """float64 rotated operands [B, L, T, D] (q', k') of the padded projection."""
    P = proj.double().view(B, L, T, 2, D)
    return gp.operands(P[..., 0, :], P[..., 1, :])


def _ops_of(x, B, L, T):
    """bf16 / f32 operand tensor [rows, T, 2, D] -> float64 q', k' [B, L, T, D]."""
    x = x.double().view(B, L, T, 2, D)
    return x[..., 0, :], x[..., 1, :]


# --------------------------------------------------------------------------- targets
@pytest.mark.parametrize("B,T,L", [(12, 3, 40), (6, 10, 64), (8, 32, 24)])
def test_targets_bit_exact(B, T, L):
    labels = _labels(B, L, T, seed=B + T)
    lens = _lens(B, L, seed=L)
    got = ops.gp_targets(_t(labels), _t(lens), _t(TYPE_TAG(T), torch.int32))
    np.testing.assert_array_equal(got.cpu().numpy(), gp.targets(labels, lens, TYPE_TAG(T)))


# --------------------------------------------------------------------------- RoPE
@pytest.mark.parametrize("B,T,L", [(3, 1, 7), (4, 3, 512)])
def test_rope_against_float64(B, T, L):
    proj, _, _ = _case(B, T, L, seed=3, scale=2.0)
    hi, lo = ops.gp_rope(proj, B, L, T, split=True)
    hi2, none = ops.gp_rope(proj, B, L, T)
    assert none is None and torch.equal(hi, hi2)
    q64, k64 = _rot64(proj, B, L, T)
    ref = torch.stack([q64, k64], 3)                                         # [B, L, T, 2, D]
    got = (hi.double() + lo.double()).view(B, L, T, 2, D)
    scale = ref.abs().max().item()
    excess = ((got - ref).abs() - 2.0 ** -16 * ref.abs()).max().item()
    print(f"rope B={B} T={T} L={L}: max(|hi + lo - ref| - 2^-16 |ref|) = {excess:.2e} (scale {scale:.2f})")
    assert excess <= 1e-6 * scale
    d = torch.randn(B * L, T, 2, D, device='cuda')
    dp = ops.gp_rope_bwd(d, B, L)
    pos = np.arange(L)
    dd = d.double().view(B, L, T, 2, D)
    ref_q = gp.rope(dd[..., 0, :], -pos) / 8.0
    ref_k = gp.rope(dd[..., 1, :], -pos)
    ref_b = torch.stack([ref_q, ref_k], 3).view(B * L, T * 2 * D)
    err = (dp.double() - ref_b).abs().max().item()
    print(f"rope bwd: max err {err:.2e}")
    assert err <= 1e-6 * ref_b.abs().max().item()


# --------------------------------------------------------------------------- loss
SHAPES = [(3, 1, 7), (64, 3, 128), (16, 10, 512)]


@pytest.mark.parametrize("B,T,L", SHAPES)
def test_loss_forward_against_float64(B, T, L):
    proj, lens, labels = _case(B, T, L, seed=B * T + L)
    sl = _t(lens)
    span_end = ops.gp_targets(_t(labels), sl, _t(TYPE_TAG(T), torch.int32))
    se = span_end.cpu().numpy()
    hi, lo = ops.gp_rope(proj, B, L, T, split=True)
    loss, lse = ops.gp_loss_fwd(hi, None, sl, span_end, L)
    ref = gp.loss(gp.scores(*_ops_of(hi, B, L, T)), se, lens).item()
    rel = abs(float(loss) - ref) / abs(ref)
    ln, lp = gp.lse(gp.scores(*_ops_of(hi, B, L, T)), se, lens)
    lse_err = (lse.double() - torch.stack([ln, lp], -1)).abs().max().item()
    loss_s, _ = ops.gp_loss_fwd(hi, lo, sl, span_end, L)
    ref_s = gp.loss(gp.scores(*_ops_of(hi.double() + lo.double(), B, L, T)), se, lens).item()
    rel_s = abs(float(loss_s) - ref_s) / abs(ref_s)
    print(f"loss B={B} T={T} L={L}: {float(loss):.6f} vs {ref:.6f} (rel {rel:.1e}, lse err {lse_err:.1e}); split "
          f"{float(loss_s):.7f} vs {ref_s:.7f} (rel {rel_s:.1e})")
    assert rel <= 1e-4 and rel_s <= 1e-5
    assert lse_err <= 1e-4 * max(1.0, torch.stack([ln, lp]).abs().max().item())
    again, lse2 = ops.gp_loss_fwd(hi, None, sl, span_end, L)
    assert torch.equal(loss, again) and torch.equal(lse, lse2)


@pytest.mark.parametrize("B,T,L", [(3, 1, 7), (64, 3, 128), (4, 3, 512)])
def test_loss_backward_against_float64_autograd(B, T, L):
    proj, lens, labels = _case(B, T, L, seed=B + T + L)
    sl = _t(lens)
    span_end = ops.gp_targets(_t(labels), sl, _t(TYPE_TAG(T), torch.int32))
    hi, _ = ops.gp_rope(proj, B, L, T)
    loss, lse = ops.gp_loss_fwd(hi, None, sl, span_end, L)
    d = ops.gp_loss_bwd(hi, sl, span_end, lse, L, 0.75)
    assert torch.equal(d, ops.gp_loss_bwd(hi, sl, span_end, lse, L, 0.75))
    q, k = (x.clone().requires_grad_(True) for x in _ops_of(hi, B, L, T))
    (0.75 * gp.loss(gp.scores(q, k), span_end.cpu().numpy(), lens)).backward()
    dv = d.double().view(B, L, T, 2, D)
    for name, g, ref in (("dQ'", dv[..., 0, :], q.grad), ("dK'", dv[..., 1, :], k.grad)):
        rel = ((g - ref).norm() / ref.norm().clamp_min(1e-30)).item()
        print(f"loss bwd B={B} T={T} L={L}: {name} norm-relative error {rel:.2e}")
        assert rel <= 1e-2, name


# --------------------------------------------------------------------------- decode
def _check_decode(hi, lo, lens, T, L, cap=None, cu=None):
    cap = L if cap is None else cap
    pred, s = ops.gp_decode(hi, lo, _t(lens), _t(TYPE_TAG(T), torch.int32), 1, 8, 9, L, cu, cap=cap, want_scores=True)
    s = s.cpu().numpy().copy()
    ref_pred, words, probs, counts = gp.decode(s, lens, TYPE_TAG(T), 1, 8, 9, cap)
    np.testing.assert_array_equal(pred.span_counts.cpu().numpy(), counts)
    np.testing.assert_array_equal(pred.cpu().numpy(), ref_pred)
    gw, gpb = pred.spans.cpu().numpy(), pred.span_probs.cpu().numpy()
    np.testing.assert_array_equal(gw, words)
    np.testing.assert_allclose(gpb, probs, rtol=2.4e-7, atol=0)
    return pred, s, counts


@pytest.mark.parametrize("B,T,L", [(8, 3, 40), (64, 3, 128), (4, 32, 24)])
def test_decode_matches_restatement(B, T, L):
    proj, lens, _ = _case(B, T, L, seed=B * T + L, scale=0.5)
    hi, lo = ops.gp_rope(proj, B, L, T, split=True)
    pred, s, counts = _check_decode(hi, None, lens, T, L)
    assert counts.sum() > 0
    pred2, s2, _ = _check_decode(hi, None, lens, T, L)
    assert torch.equal(pred, pred2) and torch.equal(pred.spans, pred2.spans)
    cand = gp.candidates(lens, L)[:, None].repeat(T, 1)
    ref = gp.scores(*_ops_of(hi, B, L, T)).cpu().numpy()
    assert np.abs(s - ref)[cand].max() <= 1e-4 * np.abs(ref[cand]).max()
    # split mode: the decode of its own s, and the sign of s against float64 wherever |s| > 1e-4
    _, ss, _ = _check_decode(hi, lo, lens, T, L)
    r64 = gp.scores(*_rot64(proj, B, L, T)).cpu().numpy()
    sure = cand & (np.abs(r64) > 1e-4)
    assert ((ss > 0) == (r64 > 0))[sure].all()


def test_decode_crafted_nesting_and_cap():
    L, T = 10, 2
    rot = torch.zeros(L, T, 2, D)
    rot[:, :, 0, 63] = 1.0                                                  # every q' . k' starts at -1 ...
    rot[:, :, 1, 63] = -1.0
    for i in range(L):
        rot[i, :, 0, i] = 1.0
    rot[4, 0, 1, 1] = 3.0                                                   # ... type 0 (1, 4): s = 2
    rot[3, 1, 1, 2] = 4.0                                                   # type 1 (2, 3): s = 3, nested in (1, 4)
    rot[4, 1, 1, 1] = 1.5                                                   # type 1 (1, 4): s = 0.5, same start as type 0
    hi = rot.to(torch.bfloat16).cuda()
    pred, s, counts = _check_decode(hi, None, np.array([9], np.int32), T, L, cap=2)
    assert counts.tolist() == [3]                                           # one more than cap: counted, not stored
    assert pred.spans.cpu().tolist() == [[1 | 5 << 12, 1 | 5 << 12 | 1 << 24]]
    assert pred.cpu().tolist() == [[8, 1, 4, 5, 1, 1, 1, 1, 9, 0]]          # the best span (2, 3) wins
    full = ops.gp_decode(hi, None, _t(np.array([9], np.int32)), _t(TYPE_TAG(T), torch.int32), 1, 8, 9, L)
    assert full.spans[0, :3].cpu().tolist() == [1 | 5 << 12, 1 | 5 << 12 | 1 << 24, 2 | 4 << 12 | 1 << 24]


def test_packed_and_padded_rows_are_bit_identical():
    B, T, L = 16, 3, 128
    proj, lens, labels = _case(B, T, L, seed=11)
    sl = _t(lens)
    keep = torch.from_numpy(np.concatenate([b * L + np.arange(n) for b, n in enumerate(lens)])).cuda()
    cu = _t(np.concatenate([[0], np.cumsum(lens)]).astype(np.int32))
    packed = proj[keep].contiguous()
    span_end = ops.gp_targets(_t(labels), sl, _t(TYPE_TAG(T), torch.int32))
    for split in (False, True):
        hp, lp = ops.gp_rope(proj, B, L, T, split=split)
        hk, lk = ops.gp_rope(packed, B, L, T, cu, split=split)
        assert torch.equal(hp[keep], hk)
        loss_p, lse_p = ops.gp_loss_fwd(hp, lp, sl, span_end, L)
        loss_k, lse_k = ops.gp_loss_fwd(hk, lk, sl, span_end, L, cu)
        assert torch.equal(loss_p, loss_k) and torch.equal(lse_p, lse_k)
        pp, sp = ops.gp_decode(hp, lp, sl, _t(TYPE_TAG(T), torch.int32), 1, 8, 9, L, want_scores=True)
        sp = sp.clone()
        pk, sk = ops.gp_decode(hk, lk, sl, _t(TYPE_TAG(T), torch.int32), 1, 8, 9, L, cu, want_scores=True)
        cand = torch.from_numpy(gp.candidates(lens, L)).cuda()[:, None].expand(B, T, L, L)
        assert torch.equal(sp[cand], sk[cand])
        assert torch.equal(pp, pk) and torch.equal(pp.spans, pk.spans) and torch.equal(pp.span_counts, pk.span_counts)
    dp = ops.gp_loss_bwd(hp, sl, span_end, lse_p, L)
    dk = ops.gp_loss_bwd(hk, sl, span_end, lse_k, L, 1.0, cu)
    assert torch.equal(dp[keep], dk)
    assert torch.equal(ops.gp_rope_bwd(dp, B, L)[keep], ops.gp_rope_bwd(dk, B, L, cu))


# --------------------------------------------------------------------------- plugin
def _estimator(tmp_path, B, L, seed, **extra):
    (tmp_path / "bert_config.json").write_text(json.dumps(SMALL_BERT))
    feats = synthetic.msra_batch(B, L, vocab=SMALL_BERT['vocab_size'], seed=seed)
    est = engine.Estimator("bert_global_pointer", dict(synthetic.data_params(L), pretrain_dir=str(tmp_path), **extra))
    est.evaluate(feats)                                                     # creates the variables
    est.store.vars["global_pointer_logits/kernel"].mul_(4.0)
    est.store.touch()
    return est, feats


def _cuda_operands(est, dev):
    """The plugin's rotated operands, by the same calls as build_graph."""
    from chinesener_b200.model import _blocks, bert_global_pointer as bgp
    from chinesener_b200.tools import layer
    table = mrc.type_table(est.params)
    B, L = dev['token_ids'].shape
    with est._layer_settings(dev), variables.use_store(est.store):
        hidden = _blocks.bert_sequence(dev, est.params, False)
        pack = getattr(hidden, 'pack', None)
        cu = pack.cu_seqlens if pack is not None else None
        w, b = est.store.vars["global_pointer_logits/kernel"], est.store.vars["global_pointer_logits/bias"]
        proj = bgp.projection(hidden, w, b, False)
        hi, lo = ops.gp_rope(proj, B, L, table.T, cu, split=layer.BERT_PRECISION == 'fp32')
    return hi, lo, cu


def gp_restatement(w, features, table, emulate_bf16, num_layers=2):
    """BertModel -> projection (bf16 operands when emulating) -> RoPE -> scores -> loss, float64."""
    t = lambda a: torch.as_tensor(np.asarray(a))
    seq = onn.bert_encoder(w, t(features['token_ids']), t(features['mask']), t(features['segment_ids']),
                           num_layers=num_layers, num_heads=12, dtype=torch.float64, emulate_bf16=emulate_bf16)
    kernel, bias = w["global_pointer_logits/kernel"].double(), w["global_pointer_logits/bias"].double()
    q, k = gp.projection(onn._rb(seq, emulate_bf16), onn._rb(kernel, emulate_bf16), bias, table.T)
    S = gp.scores(*gp.operands(q, k))
    lens = np.asarray(features['seq_len'])
    span_end = gp.targets(np.asarray(features['label_ids']), lens, table.type_tag.tolist())
    return S, gp.loss(S, span_end, lens)


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_predict_and_eval_match_restatement(tmp_path, precision):
    B, L = 6, 48
    est, feats = _estimator(tmp_path, B, L, seed=5, bert_precision=precision)
    table = mrc.type_table(est.params)
    out = est.evaluate(feats)
    res = est.predict(feats)
    pred = res['pred_ids'].numpy()
    np.testing.assert_array_equal(out['pred_ids'].numpy(), pred)
    hi, lo, cu = _cuda_operands(est, est.to_device(feats))
    lens = feats['seq_len'].numpy()
    tt = table.type_tag.tolist()
    _, s = ops.gp_decode(hi, lo, _t(lens), table.type_tag, table.o_tag, table.cls_tag, table.sep_tag, L, cu,
                         want_scores=True)
    s = s.cpu().numpy().copy()
    ref_pred, words, probs, counts = gp.decode(s, lens, tt, table.o_tag, table.cls_tag, table.sep_tag, L)
    np.testing.assert_array_equal(pred, ref_pred)                          # the decode of the plugin's own scores
    assert counts.sum() > 0 and ((pred >= 2) & (pred <= 7)).any()
    for b, spans in enumerate(res['pred_spans']):
        assert len(spans) == min(counts[b], L)
        for (name, st, en, p), wd, pr in zip(spans, words[b], probs[b]):
            assert (st, en, table.names.index(name)) == (int(wd) & 0xFFF, (int(wd) >> 12) & 0xFFF, int(wd) >> 24)
            assert abs(p - float(pr)) <= 2.4e-7 * pr
    w = est.store.state_dict()
    S_ref, loss_ref = gp_restatement(w, feats, table, emulate_bf16=precision == 'bf16')
    cand = np.broadcast_to(gp.candidates(lens, L)[:, None], s.shape)
    scale = np.abs(S_ref.numpy()[cand]).max()
    err = np.abs(s - S_ref.numpy())[cand].max()
    print(f"bert_global_pointer {precision}: max|s - restatement| = {err:.2e} (scale {scale:.2f}); loss {out['loss']:.5f} "
          f"vs {float(loss_ref):.5f}")
    assert err < 2e-2 * scale
    assert abs(out['loss'] - float(loss_ref)) < 1e-2 * abs(float(loss_ref))
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


def _train_est(tmp_path, dropout=0.0, bert_dropout=0.0, B=4, L=32):
    cfg = dict(CFG_TRAIN, hidden_dropout_prob=bert_dropout, attention_probs_dropout_prob=bert_dropout)
    (tmp_path / "bert_config.json").write_text(json.dumps(cfg))
    feats = synthetic.msra_batch(B, L, vocab=CFG_TRAIN['vocab_size'], seed=21)
    feats['seq_len'][1] = 0                                                 # an empty sentence
    feats['mask'][1] = 0
    feats['token_ids'][1] = 0
    feats['label_ids'][1] = 0
    params = dict(synthetic.data_params(L), pretrain_dir=str(tmp_path), embedding_dropout=dropout)
    return engine.Estimator("bert_global_pointer", params), feats


@pytest.mark.parametrize("packed", [True, False])
def test_gradients_match_restatement_autograd(tmp_path, packed, monkeypatch):
    from chinesener_b200.tools import layer as _layer
    monkeypatch.setattr(_layer, "TRAIN_PACK", packed)
    est, feats = _train_est(tmp_path)
    est.evaluate(feats)
    est.store.vars["global_pointer_logits/kernel"].mul_(4.0)
    est.store.touch()
    table = mrc.type_table(est.params)
    w = est.store.state_dict()
    wd = {k: v.double().clone().requires_grad_(True) for k, v in w.items()}
    _, ref_loss = gp_restatement(wd, feats, table, emulate_bf16=False)
    ref_loss.backward()
    dev = est.to_device(feats)
    with variables.use_store(est.store), autodiff.recording(est.store) as tape:
        loss, pred = est.build_graph(dev, None, est.params, True)
        tape.backward()
    rl = float(ref_loss.detach())
    assert abs(float(loss) - rl) < 2e-2 * max(1.0, abs(rl))
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
    assert "global_pointer_logits/kernel" in worst and "global_pointer_logits/bias" in worst
    bad = {k: v for k, v in worst.items() if v > 8e-2}
    print("max relative gradient error:", max(worst.values()), "over", len(worst), "variables")
    assert not bad, bad


def test_training_reduces_loss(tmp_path):
    est, feats = _train_est(tmp_path, dropout=0.1, bert_dropout=0.1)
    est.params.update(lr=5e-5, num_train_steps=100, warmup_ratio=0.1)
    losses = [float(est.train_step(feats)) for _ in range(12)]
    print("bert_global_pointer losses:", ["%.3f" % v for v in losses])
    assert np.isfinite(losses).all(), losses
    assert losses[-1] < 0.8 * losses[0], losses


def test_driver_writes_prediction_pickle(tmp_path):
    from chinesener_b200 import main as driver
    from test_main_driver_gpu import L as DRIVER_L, _setup
    root, pre = _setup(tmp_path)
    with pytest.warns(UserWarning):                                          # no BERT checkpoint: random init
        s = driver.main(['--model_name', 'bert_global_pointer', '--data', 'msra', '--data_dir', os.path.join(root, 'msra'),
                         '--checkpoint_root', str(tmp_path / 'ckpt'), '--pretrain_dir', pre, '--epoch_size', '2',
                         '--batch_size', '4'])
    assert s['n_predict'] == 24
    path = os.path.join(root, 'msra', 'bert_global_pointer_predict.pkl')
    pred = pickle.load(open(path, 'rb'))
    assert len(pred) == 24
    assert all(p['pred_ids'].shape == (DRIVER_L,) and p['pred_ids'].dtype == np.int32 for p in pred)
    assert np.isfinite(s['entity_micro_f1'])
    from chinesener_b200.data.records import NerDataset
    idx2tag = NerDataset(os.path.join(root, 'msra'), 4, 2, 'bert_global_pointer').params['idx2tag']
    tag_rep, ent_rep = evaluation.SingleEval(path, idx2tag).gen_report()
    assert 0.0 <= ent_rep['micro avg']['f1-score'] <= 1.0


def test_infer_helper_returns_nested_spans(tmp_path):
    from chinesener_b200.data.base_preprocess import features_to_batch
    from chinesener_b200.data.tokenizer import FullTokenizer
    from chinesener_b200.inference import InferHelper, TAG2IDX
    from chinesener_b200.tools.infer_utils import span_entities
    gold = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "warmup_features.json"), encoding="utf8"))
    vocab = dict(gold["bert_vocab_subset"])
    vocab.setdefault("[UNK]", 100)
    (tmp_path / "bert_config.json").write_text(json.dumps(dict(SMALL_BERT, vocab_size=21128)))
    est = engine.Estimator("bert_global_pointer", dict(synthetic.data_params(150), pretrain_dir=str(tmp_path)))
    helper = InferHelper(150, TAG2IDX, "bert_global_pointer", FullTokenizer(vocab), estimator=est)
    text = gold["text"]
    helper.infer(text)                                                      # first call creates the variables
    est.store.vars["global_pointer_logits/kernel"].mul_(4.0)
    est.store.touch()
    texts = [text, text[:7], text[3:30], text[::2]]
    batch = [dict(e) for e in helper.infer_batch(texts)]
    feats = [dict(helper.make_feature(t)) for t in texts]
    res = est.predict(features_to_batch(feats))
    assert 'pred_spans' in res
    joined = [dict(e) for e in span_entities([f['tokens'] for f in feats], res['pred_spans'])]
    assert batch == joined and any(batch)
    spans = [(s, e) for sent in res['pred_spans'] for _, s, e, _ in sent]
    assert any(a[0] <= b[0] and b[1] <= a[1] and a != b for a in spans for b in spans)      # nested spans are returned
    one = est.predict(features_to_batch([dict(helper.make_feature(text))]))
    assert dict(helper.infer(text)) == dict(span_entities([helper.make_feature(text)['tokens']], one['pred_spans'])[0])
