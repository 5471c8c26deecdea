"""CPU: corpus records (chunking, [CLS] / [SEP], word_start), the export round trip and the pretraining driver's refusals."""
import json

import numpy as np
import pytest
import torch

from chinesener_b200 import bert, mlm, pretrain, tf_checkpoint, variables
from chinesener_b200.data import corpus, records

CHARS = [chr(0x4e00 + i) for i in range(200)]
VOCAB = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]", "##a", "ab", "a"] + CHARS


def _bert_dir(tmp_path, vocab=VOCAB, **cfg):
    d = tmp_path / "bert"
    d.mkdir(parents=True, exist_ok=True)
    (d / "vocab.txt").write_text("\n".join(vocab) + "\n", encoding="utf-8")
    c = {'vocab_size': len(vocab), 'hidden_size': 32, 'num_hidden_layers': 1, 'num_attention_heads': 1,
         'intermediate_size': 64, 'max_position_embeddings': 16, 'type_vocab_size': 2}
    c.update(cfg)
    (d / "bert_config.json").write_text(json.dumps(c))
    return d


def test_chunks_of_exactly_max_seq_len_minus_two(tmp_path):
    d = _bert_dir(tmp_path)
    src = tmp_path / "a.txt"
    src.write_text("".join(CHARS[:14]) + "\n\n" + "".join(CHARS[20:26]) + "\n", encoding="utf-8")
    n_train, n_valid = corpus.build([str(src)], str(tmp_path / "out"), str(d), 8, valid_fraction=0.0)
    assert (n_train, n_valid) == (4, 0)                       # 14 = 6 + 6 + 2 pieces, then 6: blank line skipped
    rec = records.RecordFile(str(tmp_path / "out" / "train.nerrec"))
    b = rec.batch(slice(0, 4), with_strings=False)
    assert b['seq_len'].tolist() == [8, 8, 4, 8]
    ids = b['token_ids'].numpy()
    vocab = {t: i for i, t in enumerate(VOCAB)}
    for r, n in enumerate(b['seq_len'].tolist()):
        assert ids[r, 0] == vocab["[CLS]"] and ids[r, n - 1] == vocab["[SEP]"] and (ids[r, n:] == 0).all()
        assert b['mask'][r].tolist() == [1] * n + [0] * (8 - n) and not b['segment_ids'][r].any()
    assert ids[0, 1:7].tolist() == [vocab[c] for c in CHARS[:6]] and ids[2, 1:3].tolist() == [vocab[c] for c in CHARS[12:14]]


def test_word_start_from_a_segmenter(tmp_path):
    d = _bert_dir(tmp_path)
    text = CHARS[0] + CHARS[1] + CHARS[2] + "ab" + CHARS[3]           # pieces: c0 c1 c2 ab c3
    cut = lambda s: [s[0:2], s[2:4], s[4:5], s[5:6]]                   # words c0c1 | c2a | b | c3: 'ab' swallows b's start
    tok = corpus.FullTokenizer(str(d / "vocab.txt"))
    pieces, flags = corpus.tokenize_passage(tok, text, cut)
    assert pieces == [CHARS[0], CHARS[1], CHARS[2], "ab", CHARS[3]] and flags == [1, 0, 1, 0, 1]
    pieces, flags = corpus.tokenize_passage(tok, "aa", lambda s: ["a", "a"])
    assert pieces == ["a", "##a"] and flags == [1, 0]                   # ## pieces never start a word
    src = tmp_path / "b.txt"
    src.write_text(text + "\n" + text + "\n", encoding="utf-8")
    corpus.build([str(src)], str(tmp_path / "o"), str(d), 16, cut=cut, valid_fraction=0.5)
    for split in ("train", "valid"):
        b = records.RecordFile(str(tmp_path / "o" / f"{split}.nerrec")).batch(slice(0, 1), with_strings=False)
        assert b['word_start'][0].tolist() == [0, 1, 0, 1, 0, 1, 0] + [0] * 9


def test_export_round_trip(tmp_path):
    d = _bert_dir(tmp_path)
    cfg = bert.load_bert_config(str(d))
    store = variables.VariableStore('cpu', seed=9)
    with pytest.warns(UserWarning):
        bert.create_bert_variables(cfg, store)
        mlm.create_head_variables(cfg, store)
    out = tmp_path / "export"
    prefix = mlm.export_pretrained(store, str(out), str(d))
    got = tf_checkpoint.load_tf_checkpoint(prefix)
    want = {n for n in store.vars if n.startswith("bert/") or n.startswith("cls/predictions/")}
    assert set(got) == want and "bert/pooler/dense/kernel" in want and "cls/predictions/output_bias" in want
    for n in want:
        assert np.array_equal(got[n], store.vars[n].numpy()), n
    assert (out / "vocab.txt").read_text(encoding="utf-8") == (d / "vocab.txt").read_text(encoding="utf-8")
    assert json.loads((out / "bert_config.json").read_text()) == json.loads((d / "bert_config.json").read_text())
    # the head loads back through load_bert_checkpoint(scope="cls")
    other = variables.VariableStore('cpu', seed=10)
    cfg2 = bert.load_bert_config(str(out))
    bert.create_bert_variables(cfg2, other)
    mlm.create_head_variables(cfg2, other)
    for n in want:
        assert torch.equal(other.vars[n], store.vars[n]), n


def _args(tmp_path, d, **kw):
    a = {"--data_dir": str(tmp_path / "data"), "--pretrain_dir": str(d), "--output_dir": str(tmp_path / "run")}
    a.update(kw)
    return [x for kv in a.items() for x in kv]


def _data(tmp_path, d, L=8):
    src = tmp_path / "c.txt"
    src.write_text("".join(CHARS[:30]) + "\n", encoding="utf-8")
    corpus.build([str(src)], str(tmp_path / "data"), str(d), L, valid_fraction=0.2)


@pytest.mark.parametrize("flag,value,match", [("--masked_lm_prob", "0", "masked_lm_prob"), ("--masked_lm_prob", "1.5", "masked_lm_prob"),
                                              ("--max_predictions_per_seq", "0", "max_predictions_per_seq")])
def test_driver_refuses_bad_settings(tmp_path, flag, value, match):
    d = _bert_dir(tmp_path)
    _data(tmp_path, d)
    with pytest.raises(ValueError, match=match):
        pretrain.main(_args(tmp_path, d, **{flag: value}))


def test_driver_refuses_bad_vocabularies_and_lengths(tmp_path):
    d = _bert_dir(tmp_path)
    _data(tmp_path, d, L=16)
    d2 = _bert_dir(tmp_path / "x", max_position_embeddings=12)
    with pytest.raises(ValueError, match="max_position_embeddings"):
        pretrain.main(_args(tmp_path, d2))
    d3 = _bert_dir(tmp_path / "y", vocab_size=len(VOCAB) + 1)
    with pytest.raises(ValueError, match="vocab_size"):
        pretrain.main(_args(tmp_path, d3))
    d4 = _bert_dir(tmp_path / "z", vocab=[v for v in VOCAB if v != "[MASK]"])
    with pytest.raises(ValueError, match=r"\[MASK\]"):
        pretrain.main(_args(tmp_path, d4))
    big = ["[PAD]", "[MASK]"] + ["t%d" % i for i in range(50000)]
    d5 = _bert_dir(tmp_path / "w", vocab=big)
    with pytest.raises(ValueError, match="50000"):
        pretrain.main(_args(tmp_path, d5))
