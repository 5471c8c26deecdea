"""ner_featurize_wordpiece / ner_featurize_chars against the host featuriser, and InferHelper.infer_batch on the device
featuriser against infer()."""
import random

import numpy as np
import pytest
import torch

from chinesener_b200 import engine, synthetic
from chinesener_b200.data.base_preprocess import BasicProc, features_to_batch
from chinesener_b200.data.device_featurize import DeviceFeaturizer
from chinesener_b200.data.tokenizer import FullTokenizer, TokenizerAdapter, TokenizerBert, TokenizerGiga
from chinesener_b200.inference import TAG2IDX, InferHelper

pytestmark = pytest.mark.gpu

SPECIAL = ['[PAD]', '[UNK]', '[CLS]', '[SEP]', '[MASK]']
CJK = [chr(0x4E00 + i) for i in range(0, 3000, 2)]
LATIN = list('abcdefghijklmnopqrstuvwxyzABCDEFGHIJ0123456789')


def _wordpiece_vocab():
    words = ['the', 'un', '##aff', '##able', 'aff', 'able', 'run', '##ning', '##s', 'σας', 'ας', 'ς', 'a〮', '##𝅥',
             'über', 'uber', '##e', 'x', '##y', '##yz', 'ab', '##c', '\u1112', '##\u1112', '##\u1161', '##\u11ab']
    toks = SPECIAL + CJK + LATIN + ['##' + c for c in LATIN] + words + list('，。、；：！？（）,.!?-#') + ['ΑΣ', 'ασ']
    toks += ['中', 'un']                       # duplicated lines: the later line's id wins, as load_vocab does
    vocab = {}
    for i, t in enumerate(toks):
        vocab[t] = i
    return vocab


def _cursor_of(tokens):
    """fix_tokens' cursor at every [UNK] (-1 elsewhere), from the host token list."""
    out, cursor = [], 0
    for tok in tokens:
        if tok in ('[PAD]', '[CLS]', '[SEP]'):
            out.append(-1)
        elif tok == '[UNK]':
            out.append(cursor)
            cursor += 1
        else:
            out.append(-1)
            cursor += len(tok.replace('##', '') if tok.startswith('##') else tok)
    return out


def _compare(tokenizer, kind, texts, L):
    proc = BasicProc(kind, L, TAG2IDX, tokenizer)
    feats = [proc.build_seq_feature(t) for t in texts]
    want = features_to_batch(feats)
    got = DeviceFeaturizer(tokenizer, L).featurize(texts)
    torch.cuda.synchronize()
    for k in ('token_ids', 'mask', 'segment_ids', 'seq_len', 'label_ids'):
        g, w = got[k].cpu(), want[k]
        if not torch.equal(g, w):
            bad = int((g != w).reshape(len(texts), -1).any(1).nonzero()[0, 0])
            raise AssertionError(f'{k} differs for text {texts[bad]!r}: {g[bad].tolist()} != {w[bad].tolist()}')
    assert np.array_equal(got['mask'].row_lengths, want['seq_len'].numpy())
    cur = got['unk_cursor'].cpu().numpy()
    if kind == TokenizerBert:
        want_cur = np.array([_cursor_of(f['tokens']) for f in feats], dtype=np.int32).reshape(len(texts), L)
        bad = np.nonzero((cur != want_cur).any(1))[0]
        assert len(bad) == 0, (texts[bad[0]], cur[bad[0]], want_cur[bad[0]])
    else:
        unk = np.array([[t == '[UNK]' for t in f['tokens']] for f in feats]).reshape(len(texts), L)
        assert np.array_equal(cur >= 0, unk)


def _giga():
    words = CJK + LATIN + list('，。!?A') + ['中国', '[PAD]'] + CJK[:40]       # repeated words, a multi-character word
    return TokenizerAdapter(words)


TRICKY = ['', ' ', '\t\n 　 ', 'ΑΣ', 'ΑΣ ΑΣ', 'ΑΣα', 'ᾼΣ', 'ΑΣ́', 'ΑΣ́b', 'Σ', 'aΣ.b',
          'a〮\U0001d165́', 'á〮\U0001d165̖', 'e͏〮́', 'İstanbul', 'Über',
          'ǅ', ' x y', '！Ａ～　中', '\ud800', 'a\udfffb', '😀', 'x' * 201,
          'x' * 200, 'x' + 'y' * 199, 'unaffable running', 'unaffablex', 'abc', 'abcz', '#ab', 'a\x00b�c\x7f',
          '中́国', 'un中aff', '（中国）。', 'run-ning', '­', 'a​b']


@pytest.mark.parametrize('lower', [True, False])
def test_wordpiece_every_code_point(lower):
    tok = FullTokenizer(_wordpiece_vocab(), do_lower_case=lower)
    cps = [c for c in range(0x110000)]
    _compare(tok, TokenizerBert, [chr(c) for c in cps], 4)
    _compare(tok, TokenizerBert, ['a' + chr(c) + '中' for c in cps], 8)


def test_chars_every_code_point():
    tok = _giga()
    _compare(tok, TokenizerGiga, [chr(c) for c in range(0x110000)], 2)
    _compare(tok, TokenizerGiga, ['a' + chr(c) + '中' for c in range(0x110000)], 4)


def _random_texts(n, seed):
    rng = random.Random(seed)
    pool = (CJK[:200] + LATIN + list('，。!? \t　 ΑΣσßİǗ〮ͅ') + ['\U0001d165', '\ud800', 'x' * 205]
            + [chr(rng.randrange(0x80, 0x3000)) for _ in range(200)])
    return [''.join(rng.choice(pool) for _ in range(rng.randrange(0, 300))) for _ in range(n)]


@pytest.mark.parametrize('L', [8, 128, 512, 4095])
def test_tricky_and_random_texts(L):
    texts = TRICKY + _random_texts(300, L)
    for lower in (True, False):
        _compare(FullTokenizer(_wordpiece_vocab(), do_lower_case=lower), TokenizerBert, texts, L)
    _compare(_giga(), TokenizerGiga, texts, L)


def test_empty_batch():
    got = DeviceFeaturizer(FullTokenizer(_wordpiece_vocab()), 16).featurize([])
    assert got['token_ids'].shape == (0, 16) and got['mask'].total_tokens == 0


# --------------------------------------------------------------------------- infer_batch
def _bert_dir(tmp_path, vocab_size):
    import json
    cfg = {'vocab_size': vocab_size, 'hidden_size': 128, 'num_hidden_layers': 1, 'num_attention_heads': 2,
           'intermediate_size': 256, 'max_position_embeddings': 512, 'type_vocab_size': 2, 'initializer_range': 0.02}
    (tmp_path / 'bert_config.json').write_text(json.dumps(cfg))
    return str(tmp_path)


def _texts():
    rng = random.Random(5)
    base = [''.join(rng.choice(CJK[:60] + LATIN[:6] + ['，', ' ', 'Über']) for _ in range(rng.randrange(1, 60)))
            for _ in range(20)]
    return base + ['中国人民', 'á中é国', '', '  ']


def _helper(tmp_path, model, tokenizer, L, scale, **params):
    if 'bert' in model:
        params['pretrain_dir'] = _bert_dir(tmp_path, max(tokenizer.vocab.values()) + 1)
    else:
        params['embedding'] = np.random.default_rng(0).standard_normal(
            (max(tokenizer.vocab2idx.values()) + 1, 16)).astype(np.float32)
    est = engine.Estimator(model, dict(synthetic.data_params(L), **params))
    helper = InferHelper(L, TAG2IDX, model, tokenizer, estimator=est)
    helper.infer('中国')
    for k, v in est.store.vars.items():
        if k.endswith('logits/kernel'):
            v.mul_(scale)
    est.store.touch()
    return helper


def _host_infer_batch(helper, texts):
    """infer_batch on make_feature's host features: the same batch, so the same PREDICT numerics."""
    from chinesener_b200.tools.infer_utils import extract_entity_device, span_entities, span_lists
    feats = [dict(helper.make_feature(t)) for t in texts]
    pred = helper.estimator.predict_device(helper.estimator.to_device(features_to_batch(feats)))
    spans = span_lists(pred)
    if spans is not None:
        return [dict(e) for e in span_entities([f['tokens'] for f in feats], spans)]
    return [dict(e) for e in extract_entity_device([f['tokens'] for f in feats], pred, helper.idx2tag)]


@pytest.mark.parametrize('model', ['bert_crf', 'bilstm_crf', 'bert_global_pointer'])
def test_infer_batch_equals_infer(tmp_path, model):
    tok = FullTokenizer(_wordpiece_vocab()) if 'bert' in model else _giga()
    helper = _helper(tmp_path, model, tok, 64, 20.0)
    texts = _texts()
    got = [dict(e) for e in helper.infer_batch(texts)]
    assert helper.featurizer is not None
    assert got == _host_infer_batch(helper, texts)
    assert sum(len(v) for e in got for v in e.values()) > 5
    # one text per call: the batch of one infer() runs
    assert [dict(e) for t in texts[:6] for e in helper.infer_batch([t])] == [dict(helper.infer(t)) for t in texts[:6]]


def test_infer_batch_document_mode(tmp_path):
    tok = FullTokenizer(_wordpiece_vocab())
    helper = _helper(tmp_path, 'bert_crf', tok, 1500, 20.0)
    rng = random.Random(1)
    text = ''.join(rng.choice(CJK[:100]) for _ in range(1400))
    assert helper.infer_batch([text])[0] == helper.infer(text)


def test_infer_batch_unk_cursor_and_index_error(tmp_path):
    tok = FullTokenizer(_wordpiece_vocab())
    helper = _helper(tmp_path, 'bert_crf', tok, 32, 20.0)
    # removed characters before an [UNK] shift the cursor: fix_tokens reads the character the cursor lands on
    for text in ('\x00\x01中龘国́龘', 'ǅ龘中国'):
        assert [dict(e) for e in helper.infer_batch([text])] == [dict(helper.infer(text))]
    # NFD splits each Hangul syllable into three jamo, so the [UNK] cursor runs past the sentence's end: both raise
    bad = '한한한한龘'
    with pytest.raises(IndexError):
        helper.infer(bad)
    with pytest.raises(IndexError):
        helper.infer_batch(['中国', bad])


def test_word_enhance_helper_keeps_the_host_path(monkeypatch):
    from chinesener_b200 import inference
    monkeypatch.setattr(inference, 'get_instance', lambda *a, **k: None)
    helper = InferHelper(32, TAG2IDX, 'bilstm_crf_softlexicon', _giga(), estimator=None)
    assert helper.word_enhance == 'softlexicon'
    called = []
    helper.make_feature = lambda t: called.append(t) or (_ for _ in ()).throw(RuntimeError('host path'))
    with pytest.raises(RuntimeError, match='host path'):
        helper.infer_batch(['中国'])
    assert called == ['中国'] and helper.featurizer is None
