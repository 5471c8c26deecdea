"""GPU: N-best CRF decoding.  ner_crf_viterbi_nbest against the numpy list Viterbi (tests/_nbest_oracle.py) bit for bit,
rank 0 against ner_crf_viterbi under every kernel plan, path probabilities from log Z, and params['crf_nbest'] through the
CRF plugins, Estimator.predict, InferHelper.infer_nbest and main.py."""
import json
import os
import pickle

import numpy as np
import pytest
import torch

from chinesener_b200 import _lib, ops

import _nbest_oracle as nb

pytestmark = pytest.mark.gpu


def _inputs(B, L, K, seed, lens=None, aligned=True):
    g = torch.Generator().manual_seed(seed)
    x = (2.0 * torch.randn((B, L, K), generator=g)).float()
    tr = torch.randn((K, K), generator=g).float()
    if lens is None:
        lens = torch.randint(1, L + 1, (B,), generator=g)
        edge = [-3, 0, 1, L]                       # negative and zero decode like length 1
        lens[:min(B, 4)] = torch.tensor(edge[:min(B, 4)])
    lens = torch.as_tensor(lens, dtype=torch.int32)
    if aligned:
        xd = x.cuda()
    else:                                          # 4 bytes past a 16-byte boundary
        flat = torch.empty((B * L * K + 1,), dtype=torch.float32, device='cuda')
        xd = flat[1:].view(B, L, K)
        xd.copy_(x)
    return x.numpy(), tr.numpy(), lens.numpy(), xd, tr.cuda(), lens.cuda()


def _run(xd, lens_d, tr_d, N):
    tags, scores, counts = ops.crf_viterbi_nbest(xd, lens_d, tr_d, N)
    return tags.cpu().numpy(), scores.cpu().numpy(), counts.cpu().numpy()


def _check(x, tr, lens, got, N, rows):
    """Bit-exact agreement with the oracle on `rows`, plus the properties every row must have."""
    tags, scores, counts = got
    B, L, K = x.shape
    n = np.clip(lens, 1, L)
    want = np.minimum(N, np.power(float(K), np.minimum(n, 64))).astype(np.int64)
    assert np.array_equal(counts, want)
    for b in range(B):
        c = counts[b]
        assert np.all(scores[b, c:] == -np.inf) and not tags[b, c:].any()
        assert not tags[b, :, n[b]:].any()
        assert np.all(np.diff(scores[b, :c]) <= 0)
    rt, rs, rc = nb.nbest(x[rows], tr, lens[rows], N)
    assert np.array_equal(tags[rows], rt)
    assert np.array_equal(scores[rows].view(np.int32), rs.view(np.int32))
    assert np.array_equal(counts[rows], rc)
    for b in rows[:4]:
        paths = {tuple(p[:n[b]]) for p in tags[b, :counts[b]]}
        assert len(paths) == counts[b]
        for p, s in zip(tags[b, :counts[b]], scores[b, :counts[b]]):
            assert nb.path_score(x[b], tr, p[:n[b]]).view(np.int32) == np.float32(s).view(np.int32)


def _viterbi(xd, lens_d, tr_d):
    t, s = ops.crf_viterbi(xd, lens_d, tr_d, return_score=True)
    return t.cpu().numpy(), s.cpu().numpy()


KS = [1, 2, 3, 7, 10, 16, 17, 31, 32]
NS = [1, 2, 3, 8, 16]


@pytest.mark.parametrize("K", KS)
@pytest.mark.parametrize("N", NS)
def test_kernel_matches_oracle(K, N):
    B, L = 64, 128
    x, tr, lens, xd, trd, ld = _inputs(B, L, K, seed=K * 100 + N)
    got = _run(xd, ld, trd, N)
    rows = np.array(list(range(6)) + [17, 40, 63])
    _check(x, tr, lens, got, N, rows)
    vt, vs = _viterbi(xd, ld, trd)
    assert np.array_equal(got[0][:, 0], vt) and np.array_equal(got[1][:, 0].view(np.int32), vs.view(np.int32))


@pytest.mark.parametrize("L", [1, 2, 513])
@pytest.mark.parametrize("K,N", [(2, 16), (3, 3), (10, 8), (17, 2), (32, 16)])
def test_kernel_lengths(L, K, N):
    B = 64 if L < 513 else 8
    x, tr, lens, xd, trd, ld = _inputs(B, L, K, seed=L + K)
    got = _run(xd, ld, trd, N)
    _check(x, tr, lens, got, N, np.arange(min(B, 8)))
    vt, vs = _viterbi(xd, ld, trd)
    assert np.array_equal(got[0][:, 0], vt) and np.array_equal(got[1][:, 0].view(np.int32), vs.view(np.int32))


def test_document_length_rows():
    x, tr, lens, xd, trd, ld = _inputs(3, 4095, 10, seed=4095, lens=[4095, 3001, 1])
    got = _run(xd, ld, trd, 8)
    _check(x, tr, lens, got, 8, np.arange(3))


def _plan_shapes():
    """One (B, L, K, aligned) per ner_crf_viterbi plan this device reaches, chosen through ner_crf_viterbi_plan."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    cands = [(1, 128, 10, True), (64, 128, 10, True), (4500, 128, 10, True), (9000, 128, 10, True),
             (9000, 128, 10, False), (9000, 32, 17, True), (4200, 2048, 32, True), (4200, 4095, 32, True)]
    found = {}
    for B, L, K, al in cands:
        plan = _lib.VIT_PLANS[_lib.lib().ner_crf_viterbi_plan(B, L, K, int(al), sms)]
        if plan != "none":
            found.setdefault(plan, (B, L, K, al))
    return found


def test_rank0_against_every_viterbi_plan():
    found = _plan_shapes()
    assert {"small", "tma", "parked", "onchip_128", "onchip_32"} <= set(found), found
    for plan, (B, L, K, al) in found.items():
        N = 2 if L > 128 else 4
        x, tr, lens, xd, trd, ld = _inputs(B, L, K, seed=B + K, aligned=al)
        got = _run(xd, ld, trd, N)
        vt, vs = _viterbi(xd, ld, trd)
        assert np.array_equal(got[0][:, 0], vt), plan
        assert np.array_equal(got[1][:, 0].view(np.int32), vs.view(np.int32)), plan
        rows = np.unique(np.minimum([0, 1, 2, 3, B // 2, B - 1], B - 1))
        if L <= 128:
            _check(x, tr, lens, got, N, rows)
        del xd, got


def test_repeat_runs_are_bit_identical():
    x, tr, lens, xd, trd, ld = _inputs(300, 128, 10, seed=9)
    a, b = _run(xd, ld, trd, 16), _run(xd, ld, trd, 16)
    for u, v in zip(a, b):
        assert np.array_equal(u.view(np.int32), v.view(np.int32))


@pytest.mark.parametrize("L,K,N", [(2, 3, 16), (3, 2, 8), (128, 10, 8), (64, 3, 16)])
def test_probabilities_from_logz(L, K, N):
    x, tr, lens, xd, trd, ld = _inputs(64, L, K, seed=L * K)
    tags, scores, counts = ops.crf_viterbi_nbest(xd, ld, trd, N)
    logz = ops.crf_loglik_fwd(xd, tags[:, 0].contiguous(), ld, trd)[1].cpu().numpy().astype(np.float64)
    scores, counts = scores.cpu().numpy(), counts.cpu().numpy()
    n = np.clip(lens, 1, L)
    for b in range(64):
        if lens[b] <= 0:
            continue
        p = np.exp(scores[b, :counts[b]].astype(np.float64) - logz[b])
        if int(K) ** int(n[b]) <= N:                 # Python ints: K^n overflows int32
            assert abs(p.sum() - 1.0) < 1e-5, (b, p.sum())
        else:
            assert p.sum() <= 1.0 + 1e-5


# ----------------------------------------------------------------------------------------------------------- plugins
def _spy_decode(monkeypatch, plugin):
    """Record the (logits, trans, seq_len) every crf_decode of the plugin receives."""
    import importlib
    from chinesener_b200.tools import layer
    seen = []
    orig = layer.crf_decode

    def spy(logits, trans, seq_len, idx2tag, is_training, mask=None):
        seen.append((logits, trans, seq_len))
        return orig(logits, trans, seq_len, idx2tag, is_training, mask)
    monkeypatch.setattr(layer, "crf_decode", spy)
    mod = importlib.import_module("chinesener_b200.model." + plugin)
    if hasattr(mod, "crf_decode"):
        monkeypatch.setattr(mod, "crf_decode", spy)
    return seen


def _check_pred_nbest(out, base, feats, seen, n):
    assert np.array_equal(out['pred_ids'].numpy(), base['pred_ids'].numpy())        # rank 0 = the default tags
    assert 'pred_nbest' not in base
    logits, trans, seq_len = seen[-1]
    vt, vs = ops.crf_viterbi(logits, seq_len, trans, return_score=True)
    vs = vs.cpu().numpy()
    lens = feats['seq_len'].numpy()
    B, L = out['pred_ids'].shape
    K = trans.shape[0]
    assert len(out['pred_nbest']) == B
    for b, paths in enumerate(out['pred_nbest']):
        if lens[b] <= 0:
            assert paths == []
            continue
        assert len(paths) == min(n, int(K) ** min(int(lens[b]), 8))
        for tags, score, prob in paths:
            assert tags.dtype == np.int32 and tags.shape == (L,)
            assert isinstance(score, float) and 0.0 <= prob <= 1.0 + 1e-5
        assert np.array_equal(paths[0][0], out['pred_ids'][b].numpy())
        assert np.float32(paths[0][1]) == vs[b]
        assert all(a[1] >= c[1] for a, c in zip(paths, paths[1:]))


@pytest.mark.parametrize("plugin", ["bilstm_crf", "bert_crf", "bert_bilstm_crf", "lattice_lstm_crf",
                                    "transformer_crf_bichar"])
def test_plugins_nbest(plugin, tmp_path, monkeypatch):
    from test_crf_partial_gpu import _plugin
    est, feats = _plugin(plugin, tmp_path)
    est.evaluate(feats)                                   # creates the variables
    base = est.predict(feats)                             # bert_bilstm_crf: the fused executor
    seen = _spy_decode(monkeypatch, plugin)
    est.params['crf_nbest'] = 4
    out = est.predict(feats)
    assert seen, "crf_nbest > 1 must decode through build_graph"
    _check_pred_nbest(out, base, feats, seen, 4)
    ev = est.evaluate(feats)
    est.params['crf_nbest'] = 1
    ev1 = est.evaluate(feats)
    assert ev['loss'] == ev1['loss'] and np.array_equal(ev['pred_ids'].numpy(), ev1['pred_ids'].numpy())


def test_bert_bilstm_crf_document_mode_nbest(tmp_path, monkeypatch):
    from test_crf_partial_gpu import _bert_estimator
    est, feats = _bert_estimator(tmp_path, B=4, L=48)
    est.params['bert_window'] = 24
    est.evaluate(feats)
    base = est.predict(feats)
    seen = _spy_decode(monkeypatch, "bert_bilstm_crf")
    est.params['crf_nbest'] = 3
    out = est.predict(feats)
    _check_pred_nbest(out, base, feats, seen, 3)


def test_infer_nbest_first_entry_is_infer(tmp_path):
    from chinesener_b200 import engine, synthetic
    from chinesener_b200.data.tokenizer import FullTokenizer
    from chinesener_b200.inference import InferHelper, TAG2IDX
    from test_models_gpu import SMALL_BERT, _scale_up
    gold = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "warmup_features.json"), encoding="utf8"))
    vocab = dict(gold["bert_vocab_subset"])
    vocab.setdefault("[UNK]", 100)
    (tmp_path / "bert_config.json").write_text(json.dumps(dict(SMALL_BERT, vocab_size=21128)))
    est = engine.Estimator("bert_bilstm_crf", dict(synthetic.data_params(150), pretrain_dir=str(tmp_path), crf_nbest=5))
    helper = InferHelper(150, TAG2IDX, "bert_bilstm_crf", FullTokenizer(vocab), estimator=est)
    helper.infer(gold["text"])                            # first call creates the variables
    _scale_up(est.store, ["logits/kernel"], 8.0)
    cands = helper.infer_nbest(gold["text"])
    assert len(cands) == 5
    assert dict(cands[0][0]) == dict(helper.infer(gold["text"]))
    probs = [p for _, p in cands]
    assert all(a >= b for a, b in zip(probs, probs[1:])) and sum(probs) <= 1.0 + 1e-5


def test_main_driver_nbest(tmp_path):
    from chinesener_b200 import main as driver
    from test_main_driver_gpu import _setup
    root, pre = _setup(tmp_path)
    data_dir = os.path.join(root, 'msra')
    with pytest.warns(UserWarning):                       # no BERT checkpoint in pretrain_dir: random init
        s = driver.main(['--model_name', 'bert_bilstm_crf', '--data', 'msra', '--data_dir', data_dir, '--checkpoint_root',
                         str(tmp_path / 'ckpt'), '--pretrain_dir', pre, '--predict_only', '1', '--batch_size', '4',
                         '--crf_nbest', '4'])
    pred = pickle.load(open(os.path.join(data_dir, 'bert_bilstm_crf_predict.pkl'), 'rb'))
    assert len(pred) == s['n_predict'] > 0
    for p in pred:
        c = len(p['nbest_scores'])
        assert 1 <= c <= 4 and p['nbest_ids'].shape == (c, p['pred_ids'].shape[0]) and p['nbest_ids'].dtype == np.int32
        assert p['nbest_scores'].dtype == np.float32 and p['nbest_probs'].dtype == np.float32
        assert np.array_equal(p['nbest_ids'][0], p['pred_ids'])
    assert 0.0 <= s['exact_match_at_1'] <= s['exact_match_at_n'] <= 1.0
