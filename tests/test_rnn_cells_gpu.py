"""GPU: GRU cells and stacked layers of the bidirectional RNN layer (tools/layer.bilstm with cell_type / cell_size) vs
the float64 restatement of oracle/nn.py (birnn, gru_direction) and its autograd."""
import json
import os
import pickle

import numpy as np
import pytest
import torch

import _masks
import _rnn_oracle as ornn
from chinesener_b200 import autodiff, checkpoint, engine, fastpath, ops, synthetic, variables
from chinesener_b200 import main as driver
from chinesener_b200.data.tokenizer import TokenizerBert
from chinesener_b200.tools import layer, train_utils

pytestmark = pytest.mark.gpu

P = "bilstm_layer/bidirectional_rnn"
SMALL_BERT = {'vocab_size': 3000, 'hidden_size': 768, 'num_hidden_layers': 2, 'num_attention_heads': 12,
              'intermediate_size': 3072, 'max_position_embeddings': 512, 'type_vocab_size': 2, 'initializer_range': 0.02}


def _gru_w(D, H, g):
    w = {}
    lim = (6.0 / (D + 3 * H)) ** 0.5
    for d in ("fw", "bw"):
        base = f"{P}/{d}/multi_rnn_cell/cell_0/gru_cell"
        w[f"{base}/gates/kernel"] = (torch.rand(D + H, 2 * H, generator=g) * 2 - 1) * lim
        w[f"{base}/gates/bias"] = 1.0 + torch.randn(2 * H, generator=g) * 0.1
        w[f"{base}/candidate/kernel"] = (torch.rand(D + H, H, generator=g) * 2 - 1) * lim
        w[f"{base}/candidate/bias"] = torch.randn(H, generator=g) * 0.1
    return w


def _lens(B, L, g):
    lens = torch.randint(1, L + 1, (B,), generator=g, dtype=torch.int32)
    lens[0] = L
    for i, v in enumerate((0, 1, 2)):
        if i + 1 < B:
            lens[i + 1] = v
    return lens


def _rnn_masks(B, L, H, keep, seed):
    """(out, state) keep multipliers [B, L, 2H] of the recurrence kernels' DropoutWrapper (element (b, pos, dir*H + u))."""
    if keep >= 1.0:
        return None, None
    e = (np.arange(B, dtype=np.uint64)[:, None, None] * np.uint64(L) + np.arange(L, dtype=np.uint64)[None, :, None]) \
        * np.uint64(2 * H) + np.arange(2 * H, dtype=np.uint64)[None, None, :]
    lo, hi = seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF
    thr = _masks.keep_threshold(keep)
    om = _masks.hash3(lo, hi, e) < thr
    sm = _masks.hash3(lo ^ 0x5bd1e995, hi, e) < thr
    return (torch.from_numpy(om).double() / np.float32(keep), torch.from_numpy(sm).double() / np.float32(keep))


@pytest.mark.parametrize("H", [100, 128, 200, 256])
@pytest.mark.parametrize("B", [1, 7, 64, 256])
def test_gru_recurrence_matches_oracle(B, H):
    """Recurrence alone (xproj in fp64 on the host), both activations, seq_len in {0, 1, 2, L}, packed == padded."""
    L, D = 40, 24
    act = "relu" if B % 2 else "tanh"
    g = torch.Generator().manual_seed(B * 1000 + H)
    x = torch.randn(B, L, D, generator=g)
    w = _gru_w(D, H, g)
    lens = _lens(B, L, g)
    ref = ornn.birnn(x, w, lens, "gru", [H], act)
    ks = [ornn.rnn_cell_weights(w, P, d, 0, "gru") for d in ("fw", "bw")]
    xproj = torch.cat([x.double().view(B * L, D) @ k[:D] + b for k, b in ks], dim=1).float()
    whf, whb = (k[D:].float().contiguous().cuda() for k, _ in ks)
    out = ops.bigru_recurrence(xproj.cuda(), whf, whb, lens.cuda(), B, L, H, activation=act)
    torch.testing.assert_close(out.cpu().double(), ref, rtol=1e-4, atol=1e-4)
    valid = torch.arange(L)[None, :] < lens[:, None].long()
    assert (out.cpu()[~valid] == 0).all()
    cu = torch.zeros(B + 1, dtype=torch.int32)
    cu[1:] = lens.cumsum(0)
    packed = xproj.view(B, L, 6 * H)[valid].contiguous()
    outp = ops.bigru_recurrence(packed.cuda(), whf, whb, lens.cuda(), B, L, H, activation=act, cu_seqlens=cu.cuda())
    assert torch.equal(outp, out)
    assert torch.equal(ops.bigru_recurrence(xproj.cuda(), whf, whb, lens.cuda(), B, L, H, activation=act), out)


@pytest.mark.parametrize("B,L,H,act,keep", [(6, 20, 128, "tanh", 1.0), (64, 24, 128, "relu", 0.8), (5, 17, 200, "tanh", 0.7),
                                            (9, 12, 100, "relu", 0.9), (130, 8, 256, "tanh", 0.8)])
def test_gru_bptt_matches_autograd(B, L, H, act, keep):
    """d_xproj vs float64 autograd through the restatement with the kernel's dropout masks; the saved carried h and
    r * h_prev give dW_h as the caller forms it."""
    g = torch.Generator().manual_seed(B + L + H)
    seed = 0x123456789A + B
    w = _gru_w(8, H, g)
    ks = [ornn.rnn_cell_weights(w, P, d, 0, "gru")[0][8:] for d in ("fw", "bw")]    # [H, 3H] recurrent halves
    xproj = torch.randn(B * L, 6 * H, generator=g) * 0.8
    lens = _lens(B, L, g)
    om, sm = _rnn_masks(B, L, H, keep, seed)
    xp64 = xproj.double().requires_grad_(True)
    whd = [k.clone().requires_grad_(True) for k in ks]
    outs = []
    for di, rev in ((0, False), (1, True)):
        kernel = torch.cat([torch.eye(3 * H, dtype=torch.float64), whd[di]], dim=0)     # x = xproj: identity input half
        cols = slice(di * H, (di + 1) * H)
        outs.append(ornn.rnn_direction(xp64.view(B, L, 6 * H)[..., di * 3 * H:(di + 1) * 3 * H], kernel,
                                      torch.zeros(3 * H, dtype=torch.float64), lens, "gru", act, 1.0, rev, False,
                                      None if om is None else om[..., cols], None if sm is None else sm[..., cols]))
    ref = torch.cat(outs, -1)
    d_out = torch.randn(B, L, 2 * H, generator=g, dtype=torch.float64)
    (ref * d_out).sum().backward()
    whf, whb = (k.float().contiguous().cuda() for k in ks)
    out, gates, hst, rh = ops.bigru_recurrence(xproj.cuda(), whf, whb, lens.cuda(), B, L, H, activation=act,
                                               save_for_backward=True, keep_prob=keep, seed=seed)
    torch.testing.assert_close(out.cpu().double(), ref.detach(), rtol=1e-4, atol=1e-4)
    if keep == 1.0:
        assert torch.equal(hst, out)                     # carried h == emitted output without dropout
    dxp = ops.bigru_recurrence_bwd(d_out.float().cuda(), gates, hst, whf, whb, lens.cuda(), B, L, H, activation=act,
                                   keep_prob=keep, seed=seed)
    torch.testing.assert_close(dxp.cpu().double(), xp64.grad, rtol=1e-4, atol=1e-4)
    valid = torch.arange(L)[None, :] < lens[:, None].long()
    assert (dxp.cpu().view(B, L, -1)[~valid] == 0).all()
    d = dxp.cpu().double()
    hs, rhs = hst.cpu().double(), rh.cpu().double()
    for di in range(2):
        hprev = torch.zeros(B, L, H, dtype=torch.float64)
        if di == 0:
            hprev[:, 1:] = hs[:, :-1, :H]
        else:
            hprev[:, :-1] = hs[:, 1:, H:]
        dz = d[:, di * 3 * H:(di + 1) * 3 * H]
        dwg = hprev.view(B * L, H).t() @ dz[:, :2 * H]
        dwc = rhs[..., di * H:(di + 1) * H].reshape(B * L, H).t() @ dz[:, 2 * H:]
        gref = whd[di].grad
        scale = gref.abs().max().item()
        assert (torch.cat([dwg, dwc], 1) - gref).abs().max().item() < 1e-4 * max(1.0, scale)


@pytest.mark.parametrize("cell,n", [("gru", 1), ("lstm", 2), ("gru", 3)])
def test_layer_stacks_predict_and_train(cell, n):
    """tools/layer.bilstm with cell_size layers: PREDICT vs the bf16-emulated restatement; TRAIN gradients of every
    variable and of the input vs float64 autograd with the per-layer dropout masks (ragged keep probs)."""
    B, L, D = 12, 30, 50
    Hs, keeps = [128, 64, 200][:n], [0.9, 1.0, 0.8][:n]
    g = torch.Generator().manual_seed(n)
    x = torch.randn(B, L, D, generator=g) * 0.5
    lens = _lens(B, L, g)
    store = variables.VariableStore("cuda")
    with variables.use_store(store):
        out = layer.bilstm(x.cuda(), cell, "tanh", Hs, keeps, n, lens.cuda(), "float32", False)
        again = layer.bilstm(x.cuda(), cell, "tanh", Hs, keeps, n, lens.cuda(), "float32", False)
    assert torch.equal(out, again)
    w = store.state_dict()
    assert len(w) == 2 * n * (2 if cell == "lstm" else 4)
    ref = ornn.birnn(x, w, lens, cell, Hs, "tanh", emulate_bf16=True)
    err = (out.cpu().double() - ref).abs().max().item()
    print(f"{cell} x {n}: PREDICT max |out - oracle(bf16-emulated)| = {err:.2e}")
    assert err < 2e-3
    # TRAIN
    step, calls = store.global_step, store.dropout_calls
    masks = {}
    for i, (H, keep) in enumerate(zip(Hs, keeps)):
        om, sm = _rnn_masks(B, L, H, keep, (1234 * 1000003 + step) * 1009 + calls + i + 1)
        if om is not None:
            for di, d in enumerate(("fw", "bw")):
                masks[(i, d)] = (om[..., di * H:(di + 1) * H], sm[..., di * H:(di + 1) * H])
    wd = {k: v.double().requires_grad_(True) for k, v in w.items()}
    xd = x.double().requires_grad_(True)
    ref = ornn.birnn(xd, wd, lens, cell, Hs, "tanh", masks=masks)
    d_out = torch.randn(B, L, 2 * Hs[-1], generator=g, dtype=torch.float64)
    (ref * d_out).sum().backward()
    got = []
    with variables.use_store(store), autodiff.recording(store) as tape:
        xg = x.cuda()
        tape.record(xg, lambda gx: got.append(gx))
        out = layer.bilstm(xg, cell, "tanh", Hs, keeps, n, lens.cuda(), "float32", True)
        torch.testing.assert_close(out.cpu().double(), ref.detach(), rtol=0, atol=3e-2)
        tape.add_grad(out, d_out.float().cuda())
        tape.backward()
    for name, v in wd.items():
        gk, gr = store.grads[name].cpu().double(), v.grad
        scale = max(gr.abs().max().item(), 1e-6)
        assert (gk - gr).abs().max().item() < 2e-2 * scale, name
    scale = xd.grad.abs().max().item()
    assert (got[0].cpu().double() - xd.grad).abs().max().item() < 2e-2 * scale


def _plugin(model_name, tmp_path, B=8, L=32, V=3000, NW=5000, **rnn):
    feats = synthetic.msra_batch(B, L, vocab=V if model_name != "bert_bilstm_crf" else SMALL_BERT['vocab_size'], seed=4)
    g = torch.Generator().manual_seed(1)
    params = dict(synthetic.data_params(L), embedding_dropout=0.0, **rnn)
    if model_name == "bert_bilstm_crf":
        (tmp_path / "bert_config.json").write_text(json.dumps(SMALL_BERT))
        params['pretrain_dir'] = str(tmp_path)
    else:
        params['embedding'] = torch.nn.functional.normalize(torch.randn(V, 50, generator=g), dim=1).numpy()
    if model_name == "bilstm_crf_softlexicon":
        ids, wts = synthetic.softlexicon_features(B, L, NW, seed=4, lens=feats['seq_len'].numpy())
        feats['softlexicon_ids'], feats['softlexicon_weights'] = ids, wts
        params.update(word_embedding=torch.nn.functional.normalize(torch.randn(NW, 50, generator=g), dim=1).numpy(),
                      word_enhance_dim=4, max_lexicon_len=10)
    return engine.Estimator(model_name, params), feats


GRU2 = dict(cell_type='gru', cell_size=2, hidden_units_list=[128, 64], keep_prob_list=[0.8, 0.9])


@pytest.mark.parametrize("model_name", ["bilstm_crf", "bert_bilstm_crf", "bilstm_crf_softlexicon"])
def test_plugins_with_two_gru_layers(model_name, tmp_path):
    est, feats = _plugin(model_name, tmp_path, **GRU2)
    est.evaluate(feats)
    est.store.vars["logits/kernel"].mul_(6.0)
    est.store.touch()
    out = est.evaluate(feats)
    w = est.store.state_dict()
    names = [n for n in w if n.startswith(P)]
    assert sorted(names) == sorted(f"{P}/{d}/multi_rnn_cell/cell_{i}/gru_cell/{p}/{v}" for d in ("fw", "bw")
                                   for i in range(2) for p in ("gates", "candidate") for v in ("kernel", "bias"))
    assert w[f"{P}/fw/multi_rnn_cell/cell_1/gru_cell/gates/kernel"].shape == (128 + 64, 128)
    # the reference's substring LR group ('lstm' -> x100 in bert_train_op) and the AdamW bias exclusion reach them
    for n in names:
        assert 'lstm' in n and train_utils._decays(n) == n.endswith("kernel")
    p = dict(est.params, num_hidden_layers=2, num_attention_heads=12)
    ref = getattr(ornn, model_name)(w, feats, p, dtype=torch.float64, emulate_bf16=True)
    assert abs(out['loss'] - ref['loss']) < 2e-3 * max(1.0, abs(ref['loss']))
    pred = out['pred_ids'].numpy()
    assert (pred == ref['pred_ids']).mean() >= 0.99
    assert (pred[feats['mask'].numpy() == 0] == 0).all()
    # checkpoint round trip: same variables, same EVAL
    path = checkpoint.save_checkpoint(est.store, str(tmp_path / "ckpt"))
    est2, _ = _plugin(model_name, tmp_path, **GRU2)
    checkpoint.restore_checkpoint(est2.store, path)
    assert set(est2.store.vars) == set(w)
    out2 = est2.evaluate(feats)
    assert out2['loss'] == out['loss'] and np.array_equal(out2['pred_ids'].numpy(), pred)
    # a short TRAIN run brings the loss down
    losses = [float(est.train_step(feats)) for _ in range(25)]
    assert np.mean(losses[-5:]) < 0.9 * np.mean(losses[:5]), losses


def test_bert_bilstm_crf_with_a_gru_takes_build_graph(tmp_path):
    est, feats = _plugin("bert_bilstm_crf", tmp_path, cell_type='gru', cell_size=1, hidden_units_list=[128],
                         keep_prob_list=[0.8])
    first = est.predict(feats)['pred_ids']
    dev = est.to_device(feats)
    assert fastpath.bert_bilstm_crf_predict(est, dev) is None       # the fused executor is LSTM-only
    assert torch.equal(est.predict(feats)['pred_ids'], first)
    assert torch.equal(est.forward_device(dev, False)[1].cpu(), first)


def test_driver_trains_a_two_layer_gru_model(tmp_path, monkeypatch):
    from chinesener_b200.model import bert_bilstm_crf
    from test_dataset_pipeline import _prepare_two_tasks
    for k, v in GRU2.items():
        monkeypatch.setitem(bert_bilstm_crf.TRAIN_PARAMS, k, v)
    root, tok = _prepare_two_tasks(tmp_path, TokenizerBert, 64)
    cfg = dict(SMALL_BERT, vocab_size=len(tok.vocab2idx))
    pre = tmp_path / "pretrain"
    pre.mkdir()
    (pre / "bert_config.json").write_text(json.dumps(cfg))
    report = tmp_path / "rep.json"
    with pytest.warns(UserWarning):                    # no BERT checkpoint in pretrain_dir: random init
        s = driver.main(['--model_name', 'bert_bilstm_crf', '--data', 'msra', '--data_dir', os.path.join(root, 'msra'),
                         '--checkpoint_root', str(tmp_path / 'ckpt'), '--pretrain_dir', str(pre), '--epoch_size', '2',
                         '--batch_size', '4', '--report', str(report)])
    assert s['n_predict'] == 24
    pred = pickle.load(open(os.path.join(root, 'msra', 'bert_bilstm_crf_predict.pkl'), 'rb'))
    assert len(pred) == 24 and pred[0]['pred_ids'].shape == (64,)
    assert json.load(open(report))['model'] == 'bert_bilstm_crf'
    ck = checkpoint.latest_checkpoint(str(tmp_path / 'ckpt' / 'ner_msra_bert_bilstm_crf'))
    with np.load(ck) as z:
        assert f"{P}/bw/multi_rnn_cell/cell_1/gru_cell/candidate/kernel" in z.files
