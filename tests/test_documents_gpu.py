"""GPU: document mode of the BERT plugins, batches longer than the BERT window (up to 4095 tokens).

Checked here:
  * ner_window_plan against the plain restatement (oracle/windows.py) on ragged batches, bit-identical repeat calls;
  * documents that fit one window tag as the plain path does;
  * bert_crf / bert_bilstm_crf PREDICT and EVAL on documents of up to 4095 tokens against the windowed oracle (the bars of
    tests/test_long_seq_gpu.py::test_bert_bilstm_crf_predict_and_eval_at_512), in every encoder precision and mode;
  * the other supported plugins against their oracles with the windowed encoder;
  * d loss / d every variable against float64 autograd through the windowed oracle, zero gradient at unowned window rows;
  * a TRAIN run at L = 2048, PREDICT with no host synchronisation, InferHelper on a long text, and the Viterbi fallback
    for many long rows.
"""
import json

import numpy as np
import pytest
import torch

from chinesener_b200 import autodiff, bert as _bert, engine, fastpath, ops, synthetic, variables, windows
from chinesener_b200.tools import layer
from oracle import crf, models as omodels, nn as onn, windows as ow

pytestmark = pytest.mark.gpu

CFG = {'vocab_size': 1500, 'hidden_size': 768, 'num_hidden_layers': 2, 'num_attention_heads': 12,
       'intermediate_size': 3072, 'max_position_embeddings': 512, 'type_vocab_size': 2, 'initializer_range': 0.02}


# --------------------------------------------------------------------------- plan kernel
@pytest.mark.parametrize("W,S", [(512, 255), (512, 510), (128, 37), (128, 1), (3, 1)])
def test_plan_kernel_matches_restatement(W, S):
    lengths = [0, 1, 2, W, W + 1, 4095, 1300, 513, 0, 700]
    B, L = len(lengths), 4095
    g = torch.Generator().manual_seed(W + S)
    ids = torch.randint(106, 21128, (B, L), generator=g, dtype=torch.int32)
    seg = torch.randint(0, 2, (B, L), generator=g, dtype=torch.int32)
    seq_len = torch.tensor(lengths, dtype=torch.int32)
    NW, n_win = windows.window_counts(lengths, W, S)
    n_doc = sum(lengths)
    args = (ids.cuda(), seg.cuda(), seq_len.cuda(), W, S, NW, n_doc)
    a = ops.window_plan(*args, packed=True, padded=True)
    b = ops.window_plan(*args, packed=True, padded=True)
    for k in a:
        assert torch.equal(a[k], b[k]), k
    pl = ow.plan(lengths, W, S)
    pos, doc = pl['pos'], pl['doc']
    real = pos >= 0
    want_ids = np.where(real, ids.numpy()[doc[:, None], np.maximum(pos, 0)], 0)
    want_seg = np.where(real, seg.numpy()[doc[:, None], np.maximum(pos, 0)], 0)
    np.testing.assert_array_equal(a['ids'].cpu().numpy(), want_ids)
    np.testing.assert_array_equal(a['segment_ids'].cpu().numpy(), want_seg)
    np.testing.assert_array_equal(a['mask'].cpu().numpy(), real.astype(np.int32))
    np.testing.assert_array_equal(a['doc_src_padded'].cpu().numpy(), pl['src_padded'])
    np.testing.assert_array_equal(a['doc_src_packed'].cpu().numpy(), pl['src_packed'])
    assert int(a['mask'].sum()) == n_win


def test_plan_kernel_clears_windows_past_the_plan():
    lengths = [700, 3]
    W, S = 512, 255
    NW, _ = windows.window_counts(lengths, W, S)
    ids = torch.full((2, 700), 7, dtype=torch.int32, device='cuda')
    out = ops.window_plan(ids, None, torch.tensor(lengths, dtype=torch.int32, device='cuda'), W, S, NW + 2, sum(lengths),
                          packed=True)
    assert int(out['mask'][NW:].abs().sum()) == 0 and int(out['ids'][NW:].abs().sum()) == 0
    assert int(out['segment_ids'].abs().sum()) == 0                 # no segment ids: zeros


# --------------------------------------------------------------------------- plugins
def _batch(lens, L, seed=31):
    f = synthetic.msra_batch(len(lens), L, vocab=CFG['vocab_size'], seed=seed, full=True)
    for b, n in enumerate(lens):
        if n >= 1:
            f['token_ids'][b, n - 1] = 102
            f['label_ids'][b, n - 1] = 9
        for k in ('token_ids', 'label_ids', 'mask'):
            f[k][b, n:] = 0
        f['seq_len'][b] = n
    return f


def _est(tmp_path, model, lens, L, dropout=0.0, bert_dropout=0.0, **extra):
    cfg = dict(CFG, hidden_dropout_prob=bert_dropout, attention_probs_dropout_prob=bert_dropout)
    (tmp_path / "bert_config.json").write_text(json.dumps(cfg))
    params = dict(synthetic.data_params(L), pretrain_dir=str(tmp_path), embedding_dropout=dropout, **extra)
    return engine.Estimator(model, params), _batch(lens, L)


def _logits(est, dev, model):
    with est._layer_settings(dev), variables.use_store(est.store):
        emb = layer.pretrain_bert_embedding(dev['token_ids'], dev['mask'], dev['segment_ids'], est.params['pretrain_dir'],
                                            0.1, False)
        x = emb
        if model is None:
            return emb, None
        if model == "bert_bilstm_crf":
            x = layer.bilstm(emb, 'lstm', est.params['rnn_activation'], [128], [1.0], 1, dev['seq_len'], 'float32', False)
        return emb, layer.dense(x, 10, 'logits')


def test_documents_that_fit_one_window_tag_as_the_plain_path(tmp_path):
    L = 1024
    est, feats = _est(tmp_path, "bert_bilstm_crf", [512, 300, 77, 9, 1], L)
    est.evaluate(feats)
    short = {k: (v[:, :512].contiguous() if torch.is_tensor(v) and v.dim() == 2 else v) for k, v in feats.items()}
    est.store.vars["logits/kernel"].mul_(8.0)
    est.store.touch()
    pred_doc = est.predict(feats)['pred_ids']
    pred_plain = est.predict(short)['pred_ids']
    assert torch.equal(pred_doc[:, :512], pred_plain) and int(pred_doc[:, 512:].abs().sum()) == 0
    emb_doc, _ = _logits(est, est.to_device(feats), None)
    emb_plain, _ = _logits(est, est.to_device(short), None)
    assert emb_doc.shape == emb_plain.shape                           # packed rows of the same tokens
    err = (emb_doc - emb_plain).abs().max().item()
    assert err <= 2e-2 * emb_plain.abs().max().item(), err


CASES = [(512, None, [4095, 2000, 513, 300, 1], 4095), (128, 37, [1100, 513, 300, 129, 1], 1100)]


@pytest.mark.parametrize("W,S,lens,L", CASES)
@pytest.mark.parametrize("model", ["bert_crf", "bert_bilstm_crf"])
def test_long_documents_predict_and_eval(tmp_path, monkeypatch, model, W, S, lens, L):
    est, feats = _est(tmp_path, model, lens, L, bert_window=W, bert_window_stride=S)
    est.evaluate(feats)
    est.store.vars["logits/kernel"].mul_(8.0)
    est.store.touch()
    out = est.evaluate(feats)
    dev = est.to_device(feats)
    pred = est.predict_device(dev).cpu().numpy()
    np.testing.assert_array_equal(out['pred_ids'].numpy(), pred)
    _, logits = _logits(est, dev, model)
    w = est.store.state_dict()
    p = dict(est.params, num_hidden_layers=2, num_attention_heads=12)
    Wd, Sd = est.document_window()
    monkeypatch.setattr(onn, "bert_encoder", ow.windowed(Wd, Sd))
    ref = getattr(omodels, model)(w, feats, p, dtype=torch.float64, emulate_bf16=True)
    lg = logits.cpu().double()
    valid = torch.arange(L)[None, :] < feats['seq_len'][:, None]
    err = (lg - ref['logits'])[valid].abs().max().item()
    print(f"{model} W={Wd} S={Sd}: max|logit - windowed oracle(bf16-emulated)| = {err:.2e}")
    assert err < 4e-3 * max(1.0, ref['logits'][valid].abs().max().item())
    trans = w['crf_layer/transitions'].numpy()
    own, _ = crf.crf_decode(logits.cpu().numpy(), trans, feats['seq_len'].numpy(), dtype=np.float32)
    np.testing.assert_array_equal(pred, own)
    ll = crf.crf_log_likelihood(logits.cpu().numpy(), feats['label_ids'].numpy(), feats['seq_len'].numpy(), trans)
    assert abs(out['loss'] - float(np.mean(-ll))) < 1e-3 * max(1.0, abs(out['loss']))
    agree = (pred == ref['pred_ids'])[valid.numpy()].mean()
    assert agree > 0.99, agree


@pytest.mark.parametrize("mode", ["fp32", "fp8", "padded", "per_kernel"])
def test_long_documents_in_every_encoder_mode(tmp_path, monkeypatch, mode):
    lens, L = [1100, 513, 300, 1], 1100
    # fp8 with tanh cells: the ReLU cell's unbounded recurrence amplifies the encoder's rounding over 1100 steps, and the
    # fp8 tags would measure that rather than the encoder (tests/test_long_seq_gpu.py gives the numbers at L = 512)
    extra = dict(rnn_activation='tanh') if mode == "fp8" else {}
    est, feats = _est(tmp_path, "bert_bilstm_crf", lens, L, bert_window=256, **extra)
    est.evaluate(feats)
    est.store.vars["logits/kernel"].mul_(8.0)
    est.store.touch()
    base = est.evaluate(feats)
    if mode in ("fp32", "fp8"):
        est.params['bert_precision'] = mode
    else:
        monkeypatch.setattr(layer, "PACK_SEQUENCES", False) if mode == "padded" else monkeypatch.setattr(_bert, "PER_KERNEL", True)
    out = est.evaluate(feats)
    valid = (torch.arange(L)[None, :] < feats['seq_len'][:, None]).numpy()
    agree = (out['pred_ids'].numpy() == base['pred_ids'].numpy())[valid].mean()
    print(mode, "pred_ids agreement with bf16:", agree)
    # fp8 moves the logits of these random weights by more than their Viterbi margins (96.3 % on an H100); its encoder
    # accuracy is pinned by tests/test_fp8_gpu.py
    assert agree > (0.95 if mode == "fp8" else 0.99), agree
    assert np.isfinite(out['loss'])
    if mode == "fp32":
        w = est.store.state_dict()
        monkeypatch.setattr(onn, "bert_encoder", ow.windowed(256, 127))
        ref = omodels.bert_bilstm_crf(w, feats, dict(est.params, num_hidden_layers=2, num_attention_heads=12),
                                      dtype=torch.float64)
        assert abs(out['loss'] - ref['loss']) < 1e-3 * max(1.0, abs(ref['loss']))
    if mode in ("padded", "per_kernel"):
        assert abs(out['loss'] - base['loss']) < 1e-3 * max(1.0, abs(base['loss']))


def test_other_plugins_in_document_mode(tmp_path, monkeypatch):
    from test_models_gpu import _adv_setup, _bert_softlex_setup, _mtl_setup
    L, W = 700, 128
    monkeypatch.setattr(onn, "bert_encoder", ow.windowed(W, (W - 2) // 2))
    for name, setup, scale in (("softlexicon", lambda d: _bert_softlex_setup(d, B=4, L=L), ["logits/kernel"]),
                               ("mtl", lambda d: _mtl_setup(d, True, B=6, L=L), ["msra/logits/kernel", "cws/logits/kernel"]),
                               ("adv", lambda d: _adv_setup(d), None)):
        d = tmp_path / name
        d.mkdir()
        est, feats = setup(d)
        if name == "adv":                                   # _adv_setup builds L = 32 features: stretch them
            est, feats = _adv_setup(d)
            feats = _mtl_setup(d, True, B=6, L=L)[1]
            est.params['max_seq_len'] = L
            scale = ["task1_msra/logits/kernel", "task2_cws/logits/kernel", "task_discriminator/logits/kernel"]
        lens = feats['seq_len'].clone()
        lens[0] = L
        feats['seq_len'][0] = L
        feats['mask'][0] = 1
        feats['token_ids'][0, 1:L - 1] = torch.randint(106, 1500, (L - 2,), dtype=torch.int32)
        feats['token_ids'][0, L - 1] = 102
        feats['label_ids'][0, 1:L - 1] = 1
        feats['label_ids'][0, L - 1] = 9
        est.params['bert_window'] = W
        est.evaluate(feats)
        for n in scale:
            est.store.vars[n].mul_(6.0)
        est.store.touch()
        out = est.evaluate(feats)
        w = est.store.state_dict()
        p = dict(est.params, num_hidden_layers=2, num_attention_heads=12)
        ref = getattr(omodels, "bert_bilstm_crf_" + name)(w, feats, p, dtype=torch.float64, emulate_bf16=True)
        print(name, out['loss'], ref['loss'])
        assert abs(out['loss'] - ref['loss']) < 5e-3 * max(1.0, abs(ref['loss']))
        assert (out['pred_ids'].numpy() == ref['pred_ids']).mean() > 0.99
        assert torch.equal(est.predict(feats)['pred_ids'], out['pred_ids'])


# --------------------------------------------------------------------------- gradients and training
def _oracle_grads(w, feats, W, S, lstm_activation=None):
    wd = {k: v.double().clone().requires_grad_(True) for k, v in w.items()}
    seq = ow.windowed(W, S)(wd, feats['token_ids'], feats['mask'], feats['segment_ids'], num_layers=2, num_heads=12,
                            dtype=torch.float64)
    if lstm_activation is not None:
        seq = onn.bilstm(seq, wd, feats['seq_len'], lstm_activation, 1.0, torch.float64)
    logits = seq @ wd['logits/kernel'] + wd['logits/bias']
    from oracle import crf_torch
    loss = (-crf_torch.crf_log_likelihood(logits, feats['label_ids'], feats['seq_len'], wd['crf_layer/transitions'])).mean()
    loss.backward()
    return float(loss.detach()), {k: v.grad for k, v in wd.items()}


@pytest.mark.parametrize("mode", ["packed", "padded", "per_kernel"])
@pytest.mark.parametrize("model", ["bert_crf", "bert_bilstm_crf"])
def test_gradients_match_windowed_oracle_autograd(tmp_path, monkeypatch, model, mode):
    monkeypatch.setattr(layer, "TRAIN_PACK", mode == "packed")
    monkeypatch.setattr(_bert, "PER_KERNEL", mode == "per_kernel")
    W, S, lens, L = 256, 127, [1100, 300, 37], 1100
    est, feats = _est(tmp_path, model, lens, L, bert_window=W, keep_prob_list=[1.0], rnn_activation='tanh')
    est.evaluate(feats)
    est.store.vars["logits/kernel"].mul_(4.0)
    est.store.touch()
    w = est.store.state_dict()
    ref_loss, ref = _oracle_grads(w, feats, W, S, 'tanh' if model == "bert_bilstm_crf" else None)
    dev = est.to_device(feats)
    captured = {}
    fwd = _bert.bert_forward_train

    def spy(*a, **k):
        captured['win'] = fwd(*a, **k)
        return captured['win']
    monkeypatch.setattr(_bert, "bert_forward_train", spy)
    add = autodiff.Tape.add_grad

    def add_spy(tape, t, g):
        if t is captured.get('win'):
            captured['grad'] = g.clone()
        return add(tape, t, g)
    monkeypatch.setattr(autodiff.Tape, "add_grad", add_spy)
    with est._layer_settings(dev), variables.use_store(est.store), autodiff.recording(est.store) as tape:
        loss, _ = est.build_graph(dev, None, est.params, True)
        tape.backward()
    assert abs(float(loss) - ref_loss) < 2e-2 * max(1.0, abs(ref_loss))
    gscale = max(g.abs().max().item() for n, g in ref.items() if g is not None and "pooler" not in n)
    worst = {}
    for name, g_ref in ref.items():
        if g_ref is None or "pooler" in name:
            continue
        g = est.store.grads[name].cpu().double()
        worst[name] = (g - g_ref).abs().max().item() / max(g_ref.abs().max().item(), 1e-3 * gscale)
    print(model, mode, "max relative gradient error:", max(worst.values()))
    assert not {k: v for k, v in worst.items() if v > 8e-2}
    pl = ow.plan(lens, W, S)
    gw = captured['grad'].reshape(-1, CFG['hidden_size']).cpu()
    unowned = np.setdiff1d(np.arange(gw.shape[0]), pl['src_padded'])
    assert len(unowned) > 0 and int((gw[unowned] != 0).sum()) == 0
    assert bool((gw[pl['src_padded']].abs().sum(1) > 0).all())


def test_training_run_at_2048(tmp_path):
    from chinesener_b200 import checkpoint
    lens = [2048, 1500, 700, 300]
    # tanh cells: see test_gradients_match_windowed_oracle_autograd
    est, feats = _est(tmp_path, "bert_bilstm_crf", lens, 2048, dropout=0.1, bert_dropout=0.1, keep_prob_list=[0.9],
                      rnn_activation='tanh')
    est.params.update(lr=1e-5, num_train_steps=100, warmup_ratio=0.1)
    losses = [float(est.train_step(feats)) for _ in range(12)]
    print("losses:", ["%.3f" % v for v in losses])
    assert np.isfinite(losses).all() and losses[-1] < 0.8 * losses[0], losses
    before = est.evaluate(feats)
    path = checkpoint.save_checkpoint(est.store, str(tmp_path / "ckpt"), 1)
    est2, _ = _est(tmp_path, "bert_bilstm_crf", lens, 2048, keep_prob_list=[0.9], rnn_activation='tanh')
    est2.evaluate(feats)
    checkpoint.restore_checkpoint(est2.store, path)
    after = est2.evaluate(feats)
    assert torch.equal(before['pred_ids'], after['pred_ids']) and before['loss'] == after['loss']


def test_predict_has_no_host_synchronisation(tmp_path):
    est, feats = _est(tmp_path, "bert_bilstm_crf", [2000, 513, 40], 2000)
    est.predict(feats)                                     # variables, packs and workspaces exist
    dev = est.to_device(feats)
    torch.cuda.synchronize()
    assert fastpath.bert_bilstm_crf_predict(est, dev) is None
    torch.cuda.set_sync_debug_mode('error')
    try:
        pred = est.predict_device(dev)
    finally:
        torch.cuda.set_sync_debug_mode('default')
    assert torch.equal(pred, est.forward_device(dev)[1])
    short = {k: (v[:, :512].contiguous() if torch.is_tensor(v) and v.dim() == 2 else v) for k, v in feats.items()}
    short['seq_len'] = torch.clamp(feats['seq_len'], max=512)
    short['mask'] = (torch.arange(512)[None] < short['seq_len'][:, None]).to(torch.int32)
    sd = est.to_device(short)
    assert fastpath.bert_bilstm_crf_predict(est, sd) is not None


def test_infer_helper_tags_a_long_text(tmp_path):
    """~3000 characters through InferHelper: the entities read off the device tags (with the device span scan in
    infer_batch) are those extract_entity reads off a host Viterbi of the document-mode logits."""
    from chinesener_b200.data.base_preprocess import features_to_batch
    from chinesener_b200.data.tokenizer import FullTokenizer
    from chinesener_b200.inference import InferHelper, TAG2IDX
    from chinesener_b200.tools.infer_utils import extract_entity
    chars = [chr(0x4e00 + i) for i in range(600)]
    vocab = {'[PAD]': 0, '[UNK]': 100, '[CLS]': 101, '[SEP]': 102, **{c: 106 + i for i, c in enumerate(chars)}}
    rng = np.random.default_rng(3)
    text = ''.join(chars[int(i)] for i in rng.integers(0, len(chars), size=3000))
    est, _ = _est(tmp_path, "bert_bilstm_crf", [8], 3002)
    helper = InferHelper(3002, TAG2IDX, "bert_bilstm_crf", FullTokenizer(vocab), estimator=est)
    helper.infer(text)                                     # creates the variables
    est.store.vars["logits/kernel"].mul_(8.0)              # confident, varied tags: entities all along the text
    est.store.touch()
    feat = dict(helper.make_feature(text))
    dev = est.to_device(features_to_batch([feat]))
    _, logits = _logits(est, dev, "bert_bilstm_crf")
    trans = est.store.vars['crf_layer/transitions'].cpu().numpy()
    own, _ = crf.crf_decode(logits.cpu().numpy(), trans, dev['seq_len'].cpu().numpy(), dtype=np.float32)
    want = extract_entity(feat['tokens'], [int(i) for i in own[0]], helper.idx2tag)
    assert sum(len(v) for v in want.values()) > 10
    assert helper.infer(text) == want
    assert helper.infer_batch([text])[0] == want
    # with other rows in the batch the GEMMs see a different row count, so near-tie tags of these random weights may
    # round the other way: only the shape of the answer is checked there
    assert len(helper.infer_batch([text, text[:400]])) == 2


# --------------------------------------------------------------------------- Viterbi
def test_viterbi_fallback_for_many_long_rows():
    from oracle import native
    native.build()
    B, L, K = 4200, 2000, 10
    g = torch.Generator().manual_seed(11)
    logits = torch.randn(B, L, K, generator=g) * 3
    trans = torch.randn(K, K, generator=g)
    lens = torch.randint(1, L + 1, (B,), generator=g, dtype=torch.int32)
    lens[:3] = torch.tensor([L, 1, 1999], dtype=torch.int32)
    tags = ops.crf_viterbi(logits.cuda(), lens.cuda(), trans.cuda()).cpu().numpy()
    want, _ = native.crf_decode(logits.numpy(), trans.numpy(), lens.numpy())
    np.testing.assert_array_equal(tags, want)
