"""GPU: TRAIN gradients, document mode and the command-line driver on tag sets past 32 tags.

- bilstm_crf at K = 108: d loss / d every trained variable (logits/kernel, logits/bias, crf_layer/transitions and the
  BiLSTM weights, which only get a gradient through d loss / d the BiLSTM output, i.e. the projection's dx) against
  float64 autograd of oracle/nn.py + oracle/crf_torch.py.
- bert_crf in document mode at K = 108 (rows of up to 1100 tokens through the window stitching): the same against the
  float64 windowed oracle, every BERT variable included (again reached only through the projection's dx).
- bert_bilstm_crf in document mode at K = 108: PREDICT / EVAL against the windowed oracle, Viterbi bit-exact on the CUDA
  logits.
- main.py on a tiny corpus prepared with `preprocess --tag_set data` (24 entity types, 52 tags): trains, evaluates,
  writes `<model>_predict.pkl` and the entity F1 report with the data's own type names.

Tolerances, relative to each variable's largest reference gradient: past 32 tags the projection's dW is a tensor-core
GEMM on bf16 operands (fp32 accumulation), as the transformer plugins' dense_train; a bf16 operand carries 2^-9 relative
rounding, so logits/kernel is held to 2e-2.  logits/bias (an fp32 column sum) and the transitions (the fp32 CRF
backward) are held to 1e-2.  That bar is set by the 1100-step rows of document mode, where float32 alpha and beta of a
few thousand nats carry 2.4e-4 of rounding; the K-specialised kernels measure 6e-3 and 8e-3 in the same test at K = 10.  The projection's dx runs on the fp32-accurate split GEMM; the variables behind it, reached
through the bf16 recurrent / encoder GEMMs, keep the 8e-2 bar of tests/test_documents_gpu.py.
"""
import json
import os
import pickle

import numpy as np
import pytest
import torch

from chinesener_b200 import autodiff, engine, main as driver, synthetic, variables
from chinesener_b200.data import preprocess as pp
from oracle import crf, crf_torch, models as omodels, nn as onn, windows as ow

pytestmark = pytest.mark.gpu

K = 108
TYPES = ['T%02d' % i for i in range(52)]
IDX2TAG = dict(enumerate(['[PAD]', 'O'] + [p + '-' + t for t in TYPES for p in ('B', 'I')] + ['[CLS]', '[SEP]']))
CFG = {'vocab_size': 1500, 'hidden_size': 768, 'num_hidden_layers': 2, 'num_attention_heads': 12,
       'intermediate_size': 3072, 'max_position_embeddings': 512, 'type_vocab_size': 2, 'initializer_range': 0.02,
       'hidden_dropout_prob': 0.0, 'attention_probs_dropout_prob': 0.0}
TOL = {'logits/kernel': 2e-2, 'logits/bias': 1e-2, 'crf_layer/transitions': 1e-2}
TOL_OTHER = 8e-2


def _params(L, **extra):
    p = synthetic.data_params(L, label_size=K)
    p['idx2tag'] = dict(IDX2TAG)
    p['tag2idx'] = {v: k for k, v in IDX2TAG.items()}
    p.update(extra)
    return p


def _batch(lens, L, vocab, seed):
    """Rows of the given lengths ([CLS] ... [SEP]) with gold tags spread over all 108 tags."""
    f = synthetic.msra_batch(len(lens), L, vocab=vocab, seed=seed, full=True)
    rng = np.random.default_rng(seed)
    lab = rng.integers(1, K - 2, size=(len(lens), L)).astype(np.int32)
    for b, n in enumerate(lens):
        for k in ('token_ids', 'mask'):
            f[k][b, n:] = 0
        f['token_ids'][b, n - 1] = 102
        lab[b, n:] = 0
        lab[b, 0], lab[b, n - 1] = K - 2, K - 1
        f['seq_len'][b] = n
    f['label_ids'] = torch.from_numpy(lab)
    return f


def _train_grads(est, feats):
    """One TRAIN forward + backward (no optimizer step) -> (loss, {name: grad})."""
    dev = est.to_device(feats)
    for g in est.store.grads.values():
        g.zero_()
    with est._layer_settings(dev), variables.use_store(est.store), autodiff.recording(est.store) as tape:
        loss, _ = est.build_graph(dev, None, est.params, True)
        tape.backward()
    return float(loss), {n: g.detach().cpu().double() for n, g in est.store.grads.items()}


def _compare(grads, ref, label):
    """Largest error of each variable's gradient over its largest reference gradient, floored at 1e-3 of the largest
    gradient of the model (the attention key bias has an exactly-zero gradient: softmax is shift invariant), as
    tests/test_documents_gpu.py does."""
    gscale = max(g.abs().max().item() for n, g in ref.items() if g is not None and "pooler" not in n)
    worst = {}
    for name, g_ref in ref.items():
        if g_ref is None or "pooler" in name:
            continue
        g = grads[name]
        worst[name] = (g - g_ref).abs().max().item() / max(g_ref.abs().max().item(), 1e-3 * gscale)
    print(label, "relative gradient errors:", {k: "%.2e" % v for k, v in sorted(worst.items(), key=lambda kv: -kv[1])[:6]})
    for name in TOL:
        assert name in worst
    bad = {k: v for k, v in worst.items() if v > TOL.get(k, TOL_OTHER)}
    assert not bad, bad


def _crf_loss(logits, wd, feats):
    return (-crf_torch.crf_log_likelihood(logits, feats['label_ids'], feats['seq_len'], wd['crf_layer/transitions'])).mean()


def test_bilstm_crf_gradients_match_float64_autograd_at_108_tags():
    L, V = 40, 1500
    lens = [40, 33, 17, 9, 2, 40, 25, 12]
    feats = _batch(lens, L, V, seed=7)
    emb = torch.nn.functional.normalize(torch.randn(V, 50, generator=torch.Generator().manual_seed(0)), dim=1).numpy()
    est = engine.Estimator("bilstm_crf", _params(L, embedding=emb, embedding_dropout=0.0, keep_prob_list=[1.0]))
    est.evaluate(feats)
    est.store.vars["logits/kernel"].mul_(4.0)
    est.store.touch()
    loss, grads = _train_grads(est, feats)
    wd = {k: v.double().clone().requires_grad_(True) for k, v in est.store.state_dict().items()}
    x = torch.as_tensor(emb).double()[feats['token_ids'].long()]
    seq = onn.bilstm(x, wd, feats['seq_len'], 'tanh', 1.0, torch.float64)
    ref_loss = _crf_loss(seq @ wd['logits/kernel'] + wd['logits/bias'], wd, feats)
    ref_loss.backward()
    assert abs(loss - float(ref_loss)) < 2e-3 * max(1.0, abs(float(ref_loss)))
    _compare(grads, {k: v.grad for k, v in wd.items()}, "bilstm_crf K=108")


def _bert_est(tmp_path, model, L, **extra):
    (tmp_path / "bert_config.json").write_text(json.dumps(CFG))
    return engine.Estimator(model, _params(L, pretrain_dir=str(tmp_path), embedding_dropout=0.0, **extra))


def test_bert_crf_document_mode_gradients_match_float64_autograd_at_108_tags(tmp_path):
    W, S, lens, L = 256, 127, [1100, 300, 37], 1100
    feats = _batch(lens, L, CFG['vocab_size'], seed=11)
    est = _bert_est(tmp_path, "bert_crf", L, bert_window=W)
    est.evaluate(feats)
    est.store.vars["logits/kernel"].mul_(4.0)
    est.store.touch()
    loss, grads = _train_grads(est, feats)
    Wd, Sd = est.document_window()
    assert (Wd, Sd) == (W, S)
    wd = {k: v.double().clone().requires_grad_(True) for k, v in est.store.state_dict().items()}
    seq = ow.windowed(Wd, Sd)(wd, feats['token_ids'], feats['mask'], feats['segment_ids'], num_layers=2, num_heads=12,
                              dtype=torch.float64)
    ref_loss = _crf_loss(seq @ wd['logits/kernel'] + wd['logits/bias'], wd, feats)
    ref_loss.backward()
    assert abs(loss - float(ref_loss)) < 2e-2 * max(1.0, abs(float(ref_loss)))
    _compare(grads, {k: v.grad for k, v in wd.items()}, "bert_crf documents K=108")


def test_bert_bilstm_crf_document_mode_predict_and_eval_at_108_tags(tmp_path, monkeypatch):
    W, S, lens, L = 128, 37, [1100, 513, 300, 129, 1], 1100
    feats = _batch([max(n, 2) for n in lens], L, CFG['vocab_size'], seed=13)
    est = _bert_est(tmp_path, "bert_bilstm_crf", L, bert_window=W, bert_window_stride=S)
    est.evaluate(feats)
    est.store.vars["logits/kernel"].mul_(8.0)
    est.store.touch()
    out = est.evaluate(feats)
    dev = est.to_device(feats)
    pred = est.predict_device(dev).cpu().numpy()
    np.testing.assert_array_equal(out['pred_ids'].numpy(), pred)
    from chinesener_b200.tools import layer
    with est._layer_settings(dev), variables.use_store(est.store):
        emb = layer.pretrain_bert_embedding(dev['token_ids'], dev['mask'], dev['segment_ids'], est.params['pretrain_dir'],
                                            0.1, False)
        x = layer.bilstm(emb, 'lstm', est.params['rnn_activation'], [128], [1.0], 1, dev['seq_len'], 'float32', False)
        logits = layer.dense(x, K, 'logits')
    w = est.store.state_dict()
    Wd, Sd = est.document_window()
    monkeypatch.setattr(onn, "bert_encoder", ow.windowed(Wd, Sd))
    ref = omodels.bert_bilstm_crf(w, feats, dict(est.params, num_hidden_layers=2, num_attention_heads=12),
                                  dtype=torch.float64, emulate_bf16=True)
    valid = torch.arange(L)[None, :] < feats['seq_len'][:, None]
    err = (logits.cpu().double() - ref['logits'])[valid].abs().max().item()
    assert err < 4e-3 * max(1.0, ref['logits'][valid].abs().max().item()), err
    trans = w['crf_layer/transitions'].numpy()
    own, _ = crf.crf_decode(logits.cpu().numpy(), trans, feats['seq_len'].numpy(), dtype=np.float32)
    np.testing.assert_array_equal(pred, own)                          # wide Viterbi on 1100-token rows: bit-exact
    ll = crf.crf_log_likelihood(logits.cpu().numpy(), feats['label_ids'].numpy(), feats['seq_len'].numpy(), trans)
    assert abs(out['loss'] - float(np.mean(-ll))) < 1e-3 * max(1.0, abs(out['loss']))
    assert (pred == ref['pred_ids'])[valid.numpy()].mean() > 0.99


# --------------------------------------------------------------------------- main.py on a data tag set
DRIVER_TYPES = ['E%02d' % i for i in range(24)]
CHARS = [chr(0x4e00 + i) for i in range(60)]


def _corpus(src, n, seed):
    """n sentences of 6-14 characters, each with one or two entities of the 24 types (BIO), per split."""
    rng = np.random.default_rng(seed)
    sents, tags = [], []
    for _ in range(n):
        m = int(rng.integers(6, 15))
        toks = [CHARS[i] for i in rng.integers(0, len(CHARS), size=m)]
        tg = ['O'] * m
        for s in rng.choice(m - 2, size=2, replace=False):
            t = DRIVER_TYPES[int(rng.integers(0, len(DRIVER_TYPES)))]
            tg[s], tg[s + 1] = 'B-' + t, 'I-' + t
        sents.append(' '.join(toks))
        tags.append(' '.join(tg))
    return sents, tags


def test_main_trains_evaluates_and_reports_on_a_data_tag_set(tmp_path):
    src = tmp_path / 'src'
    for split, n, seed in (('train', 64, 0), ('val', 16, 1), ('test', 16, 2)):
        sents, tags = _corpus(src, n, seed)
        if split == 'train':                                          # every type appears in the train split
            for i, t in enumerate(DRIVER_TYPES):
                tags[i] = ' '.join(['B-' + t, 'I-' + t] + tags[i].split(' ')[2:])
        (src / split).mkdir(parents=True)
        (src / split / 'sentences.txt').write_text('\n'.join(sents) + '\n', encoding='utf-8')
        (src / split / 'tags.txt').write_text('\n'.join(tags) + '\n', encoding='utf-8')
    vec = tmp_path / 'chars.vec'
    rng = np.random.default_rng(5)
    vec.write_text(''.join('%s %s\n' % (c, ' '.join('%.4f' % v for v in rng.normal(size=16))) for c in CHARS),
                   encoding='utf-8')
    data = tmp_path / 'data'
    pp.main(['--src', str(src), '--out', str(data), '--tag_set', 'data', '--giga_vec', str(vec), '--max_seq_len', '24'])
    params = pickle.load(open(data / 'giga_data_params.pkl', 'rb'))
    assert params['label_size'] == 2 + 2 * len(DRIVER_TYPES) + 2 == 52
    assert params['idx2tag'][2] == 'B-E00' and params['idx2tag'][49] == 'I-E23'

    report = tmp_path / 'rep.json'
    s = driver.main(['--model_name', 'bilstm_crf', '--data', 'mini', '--data_dir', str(data), '--checkpoint_root',
                     str(tmp_path / 'ckpt'), '--epoch_size', '3', '--batch_size', '8', '--report', str(report)])
    assert s['n_predict'] == 16
    pred = pickle.load(open(data / 'bilstm_crf_predict.pkl', 'rb'))
    assert len(pred) == 16 and pred[0]['pred_ids'].shape == (24,) and int(max(p['pred_ids'].max() for p in pred)) < 52
    rep = json.load(open(report))
    assert 0.0 <= rep['entity_micro_f1'] <= 1.0 and np.isfinite(rep['tag_weighted_f1'])
    named = set(rep['entity_report']) - {'micro avg', 'macro avg', 'weighted avg'}
    assert named and named <= set(DRIVER_TYPES) and any(t > 'E07' for t in named)   # type names from data_params
    assert os.path.isdir(tmp_path / 'ckpt' / 'ner_mini_bilstm_crf')
