# -*-coding:utf-8 -*-
"""GPU: the small-table word-enhance kernels (ner_multihot_embed_fwd, ner_small_table_grad) against float64, and the
bilstm_crf_bichar / _softword / _ex_softword plugins against the oracle, float64 autograd, a short TRAIN run, the driver
and InferHelper."""
import os
import pickle

import numpy as np
import pytest
import torch

from chinesener_b200 import autodiff, engine, ops, synthetic, variables
from chinesener_b200 import main as driver
from oracle import crf_torch, nn as onn

import _word_enhance_oracle as omodels
from test_word_enhance_host import prepare_corpus, write_vec

pytestmark = pytest.mark.gpu

N_TOKS = [1, 64 * 37 + 29, 1 << 20]       # one token, a count that is no multiple of the CTA range, 2^20


def _multihot(n, V, rng):
    w = (rng.random((n, V)) < 0.3).astype(np.float32)
    w[::7] *= rng.random((len(w[::7]), V)).astype(np.float32)      # some fractional weights too
    return w


@pytest.mark.parametrize("n_tok", N_TOKS)
@pytest.mark.parametrize("V,E", [(5, 5), (8, 128), (3, 50)])
def test_multihot_embed_forward(n_tok, V, E):
    rng = np.random.default_rng(n_tok + V)
    table = rng.normal(size=(V, E)).astype(np.float32)
    w = _multihot(n_tok, V, rng)
    off, ld = 3, E + 7
    out = torch.full((n_tok, ld), 123.0, device='cuda')
    ops.multihot_embed(torch.from_numpy(table).cuda(), torch.from_numpy(w).cuda(), out=out, col_offset=off)
    got = out.cpu().numpy()
    ref = w.astype(np.float64) @ table.astype(np.float64)
    assert np.abs(got[:, off:off + E] - ref).max() <= 1e-6 * max(1.0, np.abs(ref).max())
    assert (got[:, :off] == 123.0).all() and (got[:, off + E:] == 123.0).all()          # guard columns untouched


@pytest.mark.parametrize("n_tok", N_TOKS)
@pytest.mark.parametrize("mode", ["ids", "weights"])
@pytest.mark.parametrize("V,E", [(5, 5), (8, 128)])
def test_small_table_grad(n_tok, mode, V, E):
    rng = np.random.default_rng(n_tok + E)
    off, ld = 2, E + 9
    d_out = (rng.normal(size=(n_tok, ld)) + 0.3).astype(np.float32)
    d0 = rng.normal(size=(V, E)).astype(np.float32)
    if mode == "ids":
        ids = rng.integers(-2, V + 2, n_tok).astype(np.int32)                # out-of-range ids clamp into [0, V)
        coef = np.eye(V)[np.clip(ids, 0, V - 1)]
        kw = dict(ids=torch.from_numpy(ids).cuda())
    else:
        coef = _multihot(n_tok, V, rng)
        kw = dict(weights=torch.from_numpy(coef).cuda())
    ref = d0.astype(np.float64) + coef.astype(np.float64).T @ d_out[:, off:off + E].astype(np.float64)
    dev_out = torch.from_numpy(d_out).cuda()
    grads = []
    for _ in range(2):
        d_table = torch.from_numpy(d0).cuda()
        ops.small_table_grad(d_table, dev_out, col_offset=off, **kw)
        grads.append(d_table.cpu().numpy())
    assert np.abs(grads[0] - ref).max() <= 1e-5 * np.abs(ref).max()
    assert np.array_equal(grads[0].view(np.uint32), grads[1].view(np.uint32))          # bit-identical across calls


# ----------------------------------------------------------------------------- plugins
MODELS = ["bilstm_crf_bichar", "bilstm_crf_softword", "bilstm_crf_ex_softword"]


def _setup(model_name, B=8, L=64, V=11329, NB=3000, seed=2, dropout=None, keep=None):
    feats = synthetic.msra_batch(B, L, vocab=V, seed=seed)
    rng = np.random.default_rng(seed)
    live = np.arange(L)[None, :] < feats['seq_len'].numpy()[:, None]
    feats['bichar_ids'] = torch.from_numpy(rng.integers(0, NB, (B, L)).astype(np.int32))
    feats['softword_ids'] = torch.from_numpy((rng.integers(1, 5, (B, L)) * live).astype(np.int32))
    ex = (rng.random((B, L, 5)) < 0.35).astype(np.float32)
    ex[..., 4] = ex[..., :4].sum(-1) == 0
    feats['ex_softword_ids'] = torch.from_numpy((ex * live[..., None]).reshape(B, L * 5))
    g = torch.Generator().manual_seed(0)
    emb = torch.nn.functional.normalize(torch.randn(V, 50, generator=g), dim=1).numpy()
    bemb = torch.nn.functional.normalize(torch.randn(NB, 50, generator=g), dim=1).numpy()
    params = dict(synthetic.data_params(L), embedding=emb, bichar_embedding=bemb)
    if dropout is not None:
        params.update(embedding_dropout=dropout, keep_prob_list=[keep])
    return engine.Estimator(model_name, params), feats


def _perturb_table(est):
    """Move the identity-initialised segmentation table somewhere generic so its lookup is exercised."""
    t = est.store.vars.get('word_enhance/softword_embedding')
    if t is not None:
        t.add_(torch.randn(t.shape, generator=torch.Generator().manual_seed(5)).cuda() * 0.5)
    est.store.vars['logits/kernel'].mul_(6.0)
    est.store.touch()


@pytest.mark.parametrize("model_name", MODELS)
def test_plugin_matches_oracle_at_the_bilstm_crf_bars(model_name):
    est, feats = _setup(model_name)
    est.evaluate(feats)
    _perturb_table(est)
    out = est.evaluate(feats)
    ref = getattr(omodels, model_name)(est.store.state_dict(), feats, est.params, dtype=torch.float64, emulate_bf16=True)
    assert abs(out['loss'] - ref['loss']) < 2e-3 * max(1.0, abs(ref['loss']))
    assert (out['pred_ids'].numpy() == ref['pred_ids']).mean() > 0.99
    assert (out['pred_ids'].numpy()[feats['mask'].numpy() == 0] == 0).all()
    pred = est.predict(feats)['pred_ids'].numpy()
    np.testing.assert_array_equal(pred, out['pred_ids'].numpy())


def _oracle_input(model_name, wd, feats, params):
    char = torch.as_tensor(params['embedding']).double()[feats['token_ids'].long()]
    if model_name == 'bilstm_crf_bichar':
        return torch.cat([char, torch.as_tensor(params['bichar_embedding']).double()[feats['bichar_ids'].long()]], -1)
    table = wd['word_enhance/softword_embedding']
    if model_name == 'bilstm_crf_softword':
        seg = table[feats['softword_ids'].long()]
    else:
        B, L = feats['token_ids'].shape
        seg = feats['ex_softword_ids'].double().view(B, L, 5) @ table
    return torch.cat([seg, char], -1)


@pytest.mark.parametrize("model_name", MODELS)
def test_plugin_gradients_match_oracle_autograd(model_name):
    est, feats = _setup(model_name, L=48, V=3000, dropout=0.0, keep=1.0)
    est.evaluate(feats)
    _perturb_table(est)
    w = est.store.state_dict()
    wd = {k: v.double().clone().requires_grad_(True) for k, v in w.items()}
    x = _oracle_input(model_name, wd, feats, est.params)
    lstm = onn.bilstm(x, wd, feats['seq_len'], est.params['rnn_activation'], 1.0, torch.float64)
    logits = lstm @ wd['logits/kernel'] + wd['logits/bias']
    ll = crf_torch.crf_log_likelihood(logits, feats['label_ids'], feats['seq_len'], wd['crf_layer/transitions'])
    ref_loss = (-ll).mean()
    ref_loss.backward()
    ref_loss = ref_loss.item()
    dev = est.to_device(feats)
    with variables.use_store(est.store), autodiff.recording(est.store) as tape:
        loss, _ = est.build_graph(dev, None, est.params, True)
        tape.backward()
    assert abs(float(loss) - ref_loss) < 2e-3 * max(1.0, abs(ref_loss))
    assert ('word_enhance/softword_embedding' in wd) == (model_name != 'bilstm_crf_bichar')
    for name, v in wd.items():
        g = est.store.grads[name].cpu().double()
        scale = max(v.grad.abs().max().item(), 1e-6)
        assert (g - v.grad).abs().max().item() < 2e-2 * scale, name


@pytest.mark.parametrize("model_name", MODELS)
def test_twelve_train_steps_lower_the_loss(model_name):
    est, feats = _setup(model_name, L=48, V=3000)                  # TRAIN_PARAMS dropout on
    losses = [float(est.train_step(feats)) for _ in range(12)]
    assert np.isfinite(losses).all() and losses[-1] < 0.9 * losses[0], losses


def test_driver_run_of_the_ex_softword_plugin_writes_the_prediction_pickle(tmp_path):
    out = prepare_corpus(tmp_path, 'ex_softword')
    s = driver.main(['--model_name', 'bilstm_crf_ex_softword', '--data', 'msra', '--data_dir', out,
                     '--checkpoint_root', str(tmp_path / 'ckpt'), '--epoch_size', '2', '--batch_size', '4'])
    assert s['n_predict'] == 24 and s['history']['final_step'] == 16 * 2 // 4
    pred = pickle.load(open(os.path.join(out, 'bilstm_crf_ex_softword_predict.pkl'), 'rb'))
    assert len(pred) == 24 and pred[0]['pred_ids'].shape == (150,)


@pytest.mark.parametrize("model_name", ["bilstm_crf_bichar", "transformer_tener_crf_bichar"])
def test_infer_helper_serves_text_to_the_bichar_plugins(model_name, tmp_path):
    from chinesener_b200.data.base_preprocess import features_to_batch
    from chinesener_b200.data.tokenizer import get_giga_tokenizer
    from chinesener_b200.inference import InferHelper, TAG2IDX
    from chinesener_b200.tools.infer_utils import extract_entity
    text = '中共中央致中国致公党十一大的贺词，各位代表、各位同志：在中国致公党第十一次全国代表大会隆重召开之际。'
    chars = sorted(set(text))
    tok = get_giga_tokenizer(write_vec(tmp_path / 'giga.vec', chars, dim=50))
    btok = get_giga_tokenizer(write_vec(tmp_path / 'bi.vec', sorted({text[i:i + 2] for i in range(0, len(text) - 1, 2)}), dim=50))
    params = dict(synthetic.data_params(150), embedding=tok.embedding(0), bichar_embedding=btok.embedding(1))
    est = engine.Estimator(model_name, params)
    helper = InferHelper(150, TAG2IDX, model_name, tok, estimator=est, bichar_tokenizer=btok)
    helper.infer(text)                                            # first call creates the variables
    est.store.vars['logits/kernel'].mul_(8.0)
    est.store.touch()
    ent = helper.infer(text)
    assert helper.feature['bichar_ids'][len(text) - 1] == btok.vocab2idx['[UNK]']      # '。-null-' is not in the table
    pred = est.predict(features_to_batch([helper.feature]))['pred_ids'].numpy()[0]
    assert pred[len(text):].tolist() == [0] * (150 - len(text))
    idx2tag = {v: k for k, v in TAG2IDX.items()}
    assert dict(ent) == dict(extract_entity(helper.feature['tokens'], [int(i) for i in pred], idx2tag))
