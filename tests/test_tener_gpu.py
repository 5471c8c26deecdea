"""GPU: fp32-accurate dense (split-bf16 wgmma), fp32 TENER attention and the TENER plugin vs the oracle."""
import numpy as np
import pytest
import torch

from chinesener_b200 import engine, ops, synthetic
from oracle import models as omodels, transformer as otf

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("M,K,N", [(8192, 160, 320), (1000, 100, 160), (300, 320, 160), (4096, 768, 768)])
def test_split_bf16_gemm_reaches_fp32_accuracy(M, K, N):
    g = torch.Generator().manual_seed(M + K)
    x = torch.randn(M, K, generator=g)
    w = torch.randn(K, N, generator=g) * 0.2
    b = torch.randn(N, generator=g)
    r = torch.randn(M, N, generator=g)
    Kp = (K + 7) // 8 * 8
    wp = torch.nn.functional.pad(w, (0, 0, 0, Kp - K)).cuda().contiguous()
    w_hi = ops.pack_weight_bf16(wp)
    w_lo = ops.pack_weight_bf16((wp - w_hi.float().t()).contiguous())
    a_hi, a_lo = ops.split_bf16(x.cuda(), Kp)
    torch.testing.assert_close((a_hi.float() + a_lo.float())[:, :K].cpu(), x, rtol=2e-5, atol=1e-6)
    out = ops.gemm_split_f32(a_hi, a_lo, w_hi, w_lo, b.cuda(), residual=r.cuda(), relu=True)
    ref = torch.relu(x.double() @ w.double() + b.double() + r.double())
    err = (out.cpu().double() - ref).abs().max().item()
    scale = ref.abs().max().item()
    assert err < 3e-5 * max(1.0, scale), (err, scale)


@pytest.mark.parametrize("B,L,NH,DH,rel", [(4, 64, 8, 20, True), (3, 256, 8, 20, True), (2, 150, 4, 40, True),
                                           (2, 128, 12, 64, False), (3, 33, 2, 32, False)])
def test_attention_f32(B, L, NH, DH, rel):
    g = torch.Generator().manual_seed(B * L + DH)
    d = NH * DH
    q, k, v = (torch.randn(B * L, d, generator=g) for _ in range(3))
    u = torch.randn(NH, DH, generator=g) * 0.3
    vb = torch.randn(NH, DH, generator=g) * 0.3
    lens = torch.randint(1, L + 1, (B,), generator=g, dtype=torch.int32)
    lens[0] = L
    table = torch.from_numpy(np.asarray(otf.sinusoidal_positional_encoding(DH, np.arange(-L, L)), dtype=np.float32)) if rel else None
    scale = 1.0 if rel else DH ** -0.5
    out, hi, lo = ops.attention_f32(q.cuda(), k.cuda(), v.cuda(), lens.cuda(), B, L, NH, DH, scale=scale,
                                    bias_u=u.cuda() if rel else None, bias_v=vb.cuda() if rel else None,
                                    rel_table=table.cuda() if rel else None, want_split=True)
    sh = lambda t: t.double().view(B, L, NH, DH).permute(0, 2, 1, 3)
    Q, K, V = sh(q), sh(k), sh(v)
    if rel:
        AC = torch.einsum('bnqd,bnkd->bnqk', Q + u.double()[:, None, :], K)
        BD = otf.shift(torch.einsum('bnqd,ld->bnql', Q + vb.double()[:, None, :], table.double()))
        s = AC + BD
    else:
        s = Q @ K.transpose(-1, -2) * scale
    mask = (torch.arange(L)[None, :] < lens.long()[:, None])
    s = s + (~mask)[:, None, None, :].double() * otf.MASK_ADD
    ref = (torch.softmax(s, -1) @ V).permute(0, 2, 1, 3).reshape(B, L, d)
    o = out.cpu().double().view(B, L, d)
    for b in range(B):
        n = int(lens[b])
        assert (o[b, :n] - ref[b, :n]).abs().max() < 2e-5
        assert (o[b, n:] == 0).all()
    torch.testing.assert_close((hi.float() + lo.float()).cpu(), out.cpu(), rtol=2e-5, atol=1e-6)


def test_tener_plugin_matches_oracle_at_fp32_accuracy():
    """BASELINE config 5 shape (reduced batch): logits within 1e-3 of the float64 oracle (the
    north-star tolerance for fp32 emission logits), pred_ids equal wherever margins allow."""
    B, L, V, VB = 6, 256, 3000, 5000
    feats = synthetic.msra_batch(B, L, vocab=V, seed=9)
    g = torch.Generator().manual_seed(2)
    feats['bichar_ids'] = torch.randint(0, VB, (B, L), generator=g, dtype=torch.int32)
    emb = torch.nn.functional.normalize(torch.randn(V, 50, generator=g), dim=1).numpy()
    bemb = torch.nn.functional.normalize(torch.randn(VB, 50, generator=g), dim=1).numpy()
    params = dict(synthetic.data_params(L), embedding=emb, bichar_embedding=bemb)
    est = engine.Estimator("transformer_tener_crf_bichar", params)
    est.evaluate(feats)
    est.store.vars["logits/kernel"].mul_(4.0)
    est.store.touch()
    out = est.evaluate(feats)
    w = est.store.state_dict()
    ref = omodels.transformer_tener_crf_bichar(w, feats, est.params, dtype=torch.float64)
    # emission logits through the public layer API
    from chinesener_b200 import variables
    from chinesener_b200.tools import layer
    from chinesener_b200.tools.transformer.encoder import tener_encoder
    from chinesener_b200.tools.transformer.modules import embedding_project
    dev = est.to_device(feats)
    with variables.use_store(est.store):
        e = torch.empty((B * L, 100), dtype=torch.float32, device="cuda")
        ops.embedding_lookup(torch.from_numpy(emb).cuda(), dev['token_ids'], out=e)
        ops.embedding_lookup(torch.from_numpy(bemb).cuda(), dev['bichar_ids'], out=e, col_offset=50)
        x = tener_encoder(embedding_project(e, 160).view(B, L, -1), dev['seq_len'], L, 2, 8, 0.2, 320, False)
        logits = layer.dense(x, 10, 'logits')
    valid = torch.arange(L)[None, :] < feats['seq_len'][:, None]
    err = (logits.cpu().double() - ref['logits'])[valid].abs().max().item()
    print(f"tener: max|logit - fp64 oracle| = {err:.2e} (max |logit| {ref['logits'][valid].abs().max().item():.2f})")
    assert err < 1e-3
    assert abs(out['loss'] - ref['loss']) < 1e-3 * max(1.0, abs(ref['loss']))
    agree = (out['pred_ids'].numpy() == ref['pred_ids']).mean()
    assert agree > 0.999, agree
    assert (out['pred_ids'].numpy()[feats['mask'].numpy() == 0] == 0).all()


@pytest.mark.parametrize("B,L,NH,DH,rel", [(3, 64, 8, 20, True), (2, 256, 8, 20, True), (2, 96, 4, 40, True), (2, 70, 3, 32, False)])
def test_attention_f32_backward(B, L, NH, DH, rel):
    """ner_attention_f32_bwd vs float64 autograd of the reference formulation (tener.py:12-74 via oracle.shift)."""
    g = torch.Generator().manual_seed(B * L + DH + 1)
    d = NH * DH
    q, k, v, do = (torch.randn(B * L, d, generator=g) * 0.5 for _ in range(4))
    u = torch.randn(NH, DH, generator=g) * 0.3
    vb = torch.randn(NH, DH, generator=g) * 0.3
    lens = torch.randint(1, L + 1, (B,), generator=g, dtype=torch.int32)
    lens[0] = L
    table = torch.from_numpy(np.asarray(otf.sinusoidal_positional_encoding(DH, np.arange(-L, L)), dtype=np.float32)) if rel else None
    scale = 1.0 if rel else DH ** -0.5
    qd, kd, vd, ud, vbd = (t.double().requires_grad_(True) for t in (q, k, v, u, vb))
    sh = lambda t: t.view(B, L, NH, DH).permute(0, 2, 1, 3)
    Q, K, V = sh(qd), sh(kd), sh(vd)
    if rel:
        s = torch.einsum('bnqd,bnkd->bnqk', Q + ud[:, None, :], K) + otf.shift(torch.einsum('bnqd,ld->bnql', Q + vbd[:, None, :], table.double()))
    else:
        s = Q @ K.transpose(-1, -2) * scale
    mask = (torch.arange(L)[None, :] < lens.long()[:, None])
    s = s + (~mask)[:, None, None, :].double() * otf.MASK_ADD
    out = (torch.softmax(s, -1) @ V).permute(0, 2, 1, 3).reshape(B * L, d)
    rowmask = mask.reshape(B * L, 1).double()                 # padded query rows never reach the loss
    (out * do.double() * rowmask).sum().backward()
    dq, dk, dv, du, dvb = ops.attention_f32_bwd(q.cuda(), k.cuda(), v.cuda(), lens.cuda(), B, L, NH, DH, do.cuda(), scale=scale,
                                                bias_u=u.cuda() if rel else None, bias_v=vb.cuda() if rel else None,
                                                rel_table=table.cuda() if rel else None)
    for name, got, ref in (("dq", dq, qd.grad), ("dk", dk, kd.grad), ("dv", dv, vd.grad)):
        err = (got.cpu().double() - ref).abs().max().item()
        assert err < 2e-4 * max(1.0, ref.abs().max().item()), (name, err)
    if rel:
        for name, got, ref in (("du", du, ud.grad), ("dvb", dvb, vbd.grad)):
            err = (got.cpu().double() - ref).abs().max().item()
            assert err < 5e-4 * max(1.0, ref.abs().max().item()), (name, err)


def _tener_setup(B=4, L=64, V=2000, VB=3000, drop=0.0):
    feats = synthetic.msra_batch(B, L, vocab=V, seed=19)
    g = torch.Generator().manual_seed(3)
    feats['bichar_ids'] = torch.randint(0, VB, (B, L), generator=g, dtype=torch.int32)
    emb = torch.nn.functional.normalize(torch.randn(V, 50, generator=g), dim=1).numpy()
    bemb = torch.nn.functional.normalize(torch.randn(VB, 50, generator=g), dim=1).numpy()
    params = dict(synthetic.data_params(L), embedding=emb, bichar_embedding=bemb, embedding_dropout=drop, fc_dropout=drop,
                  dropout_rate=drop)
    return engine.Estimator("transformer_tener_crf_bichar", params), feats, emb, bemb


def test_tener_gradients_match_oracle_autograd():
    """TRAIN mode of transformer_tener_crf_bichar (BASELINE config 5's model): every variable's gradient against
    float64 autograd of the oracle (bf16 operands in the gradient GEMMs: 3e-2 of each gradient's scale)."""
    from chinesener_b200 import autodiff, variables
    from oracle import crf_torch
    est, feats, emb, bemb = _tener_setup()
    est.evaluate(feats)
    w = est.store.state_dict()
    wd = {k: v.double().clone().requires_grad_(True) for k, v in w.items()}
    x = torch.cat([torch.from_numpy(emb).double()[feats['token_ids'].long()], torch.from_numpy(bemb).double()[feats['bichar_ids'].long()]], -1)
    x = x @ wd["embedding/dense/kernel"] + wd["embedding/dense/bias"]
    x = otf.tener_encoder(x, feats['seq_len'], wd, est.params['encode_layers'], est.params['num_head'])
    logits = x @ wd['logits/kernel'] + wd['logits/bias']
    ll = crf_torch.crf_log_likelihood(logits, feats['label_ids'], feats['seq_len'], wd['crf_layer/transitions'])
    ref_loss = (-ll).mean()
    ref_loss.backward()
    dev = est.to_device(feats)
    with variables.use_store(est.store), autodiff.recording(est.store) as tape:
        loss, _ = est.build_graph(dev, None, est.params, True)
        tape.backward()
    assert abs(float(loss) - float(ref_loss)) < 2e-3 * max(1.0, abs(float(ref_loss)))
    gscale = max(v.grad.abs().max().item() for v in wd.values() if v.grad is not None)
    worst = {}
    for name, v in wd.items():
        if v.grad is None:
            continue
        g = est.store.grads[name].cpu().double()
        worst[name] = (g - v.grad).abs().max().item() / max(v.grad.abs().max().item(), 1e-3 * gscale)
    bad = {k: e for k, e in worst.items() if e > 3e-2}
    print("tener max relative gradient error:", max(worst.values()), "over", len(worst), "variables")
    assert not bad, bad


def test_tener_training_reduces_the_loss():
    est, feats, _, _ = _tener_setup(drop=0.2)
    est.params.update(lr=2e-3, num_train_steps=200, warmup_ratio=0.1)
    losses = [float(est.train_step(feats)) for _ in range(40)]
    assert np.isfinite(losses).all() and losses[-1] < 0.7 * losses[0], losses


def _abs_setup(B=4, L=64, V=2000, VB=3000, drop=0.0):
    feats = synthetic.msra_batch(B, L, vocab=V, seed=23)
    g = torch.Generator().manual_seed(5)
    feats['bichar_ids'] = torch.randint(0, VB, (B, L), generator=g, dtype=torch.int32)
    emb = torch.nn.functional.normalize(torch.randn(V, 50, generator=g), dim=1).numpy()
    bemb = torch.nn.functional.normalize(torch.randn(VB, 50, generator=g), dim=1).numpy()
    params = dict(synthetic.data_params(L), embedding=emb, bichar_embedding=bemb, embedding_dropout=drop, dropout_rate=drop)
    return engine.Estimator("transformer_crf_bichar", params), feats, emb, bemb


def test_transformer_crf_bichar_plugin_matches_oracle():
    """SURVEY 8(f) rank 4: the absolute-position transformer plugin on the same kernels (logits at fp32 accuracy)."""
    est, feats, emb, bemb = _abs_setup()
    est.evaluate(feats)
    est.store.vars["logits/kernel"].mul_(4.0)
    est.store.touch()
    out = est.evaluate(feats)
    w = est.store.state_dict()
    ref = omodels.transformer_crf_bichar(w, feats, est.params, dtype=torch.float64)
    assert abs(out['loss'] - ref['loss']) < 1e-3 * max(1.0, abs(ref['loss']))
    assert (out['pred_ids'].numpy() == ref['pred_ids']).mean() > 0.995


def test_transformer_crf_bichar_gradients_and_training():
    from chinesener_b200 import autodiff, variables
    from oracle import crf_torch
    est, feats, emb, bemb = _abs_setup()
    est.evaluate(feats)
    w = est.store.state_dict()
    wd = {k: v.double().clone().requires_grad_(True) for k, v in w.items()}
    L = feats['token_ids'].shape[1]
    x = torch.cat([torch.from_numpy(emb).double()[feats['token_ids'].long()], torch.from_numpy(bemb).double()[feats['bichar_ids'].long()]], -1)
    x = x @ wd["embedding/dense/kernel"] + wd["embedding/dense/bias"]
    x = x + otf.sinusoidal_positional_encoding(160, np.arange(L), torch.float64)[None]
    x = otf.transformer_encoder(x, feats['seq_len'], wd, est.params['encode_layers'], est.params['num_head'])
    logits = x @ wd['logits/kernel'] + wd['logits/bias']
    ref_loss = (-crf_torch.crf_log_likelihood(logits, feats['label_ids'], feats['seq_len'], wd['crf_layer/transitions'])).mean()
    ref_loss.backward()
    dev = est.to_device(feats)
    with variables.use_store(est.store), autodiff.recording(est.store) as tape:
        loss, _ = est.build_graph(dev, None, est.params, True)
        tape.backward()
    assert abs(float(loss) - float(ref_loss.detach())) < 2e-3 * max(1.0, abs(float(ref_loss.detach())))
    gscale = max(v.grad.abs().max().item() for v in wd.values() if v.grad is not None)
    worst = {n: (est.store.grads[n].cpu().double() - v.grad).abs().max().item() / max(v.grad.abs().max().item(), 1e-3 * gscale)
             for n, v in wd.items() if v.grad is not None}
    assert max(worst.values()) < 3e-2, {k: e for k, e in worst.items() if e > 3e-2}
    est2, feats2, _, _ = _abs_setup(drop=0.2)
    est2.params.update(lr=2e-3, num_train_steps=200, warmup_ratio=0.1)
    losses = [float(est2.train_step(feats2)) for _ in range(40)]
    assert np.isfinite(losses).all() and losses[-1] < 0.7 * losses[0], losses
