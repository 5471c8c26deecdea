"""The device featuriser's host half (data/device_featurize.py) and the argument checks of ner_featurize_* — no GPU."""
import ctypes
import unicodedata

import numpy as np
import pytest

from chinesener_b200 import _lib
from chinesener_b200.data import device_featurize as df
from chinesener_b200.data.tokenizer import _is_chinese_char, _is_control, _is_punctuation, _is_whitespace


def test_unicode_tables_match_unicodedata_for_every_code_point():
    tables = df.unicode_tables()
    rec = df.unicode_record(tables, np.arange(df.N_CODEPOINTS))
    assert tables['stage1'].shape == (df.N_CODEPOINTS >> 8,)
    for cp in range(df.N_CODEPOINTS):
        ch, r = chr(cp), int(rec[cp])
        assert bool(r & df.F_CONTROL) == _is_control(ch), cp
        assert bool(r & df.F_WHITESPACE) == _is_whitespace(ch), cp
        assert bool(r & df.F_SPACE) == ch.isspace(), cp
        assert bool(r & df.F_PUNCT) == _is_punctuation(ch), cp
        assert bool(r & df.F_CJK) == _is_chinese_char(cp), cp
        assert bool(r & df.F_MN) == (unicodedata.category(ch) == 'Mn'), cp
        assert (r >> 8) & 0xFF == unicodedata.combining(ch), cp
        x = r >> 16
        want = unicodedata.normalize('NFD', ch.lower())
        got = ''.join(chr(c) for c in tables['expand'][x] if c) if x else ch
        assert got == want, cp
        # Final_Sigma as str.lower() applies it: after a cased letter and this character, at the end of the word
        ignorable, cased = bool(r & df.F_IGNORABLE), bool(r & df.F_CASED)
        assert (('A' + ch + 'Σ').lower()[-1] == 'ς') == (ignorable or cased), cp
        assert (('AΣ' + ch).lower()[1] == 'ς') == (ignorable or not cased), cp


def test_unicode_tables_hold_the_cases_the_kernel_relies_on():
    rec = df.unicode_record(df.unicode_tables(), [0x2028, 0x2029, 0x3000, 0x302E, 0x1D165, 0x0301, 0x3A3])
    assert rec[0] & df.F_SPACE and not rec[0] & df.F_WHITESPACE           # split on, but not Zs
    assert rec[2] & df.F_SPACE and rec[2] & df.F_WHITESPACE
    assert not rec[3] & df.F_MN and (rec[3] >> 8) & 0xFF == 224            # nonzero class, survives the Mn strip
    assert not rec[4] & df.F_MN and (rec[4] >> 8) & 0xFF == 216
    assert rec[5] & df.F_MN and (rec[5] >> 8) & 0xFF == 230
    assert rec[6] & df.F_CASED and not rec[6] & df.F_IGNORABLE


def test_vocab_table_finds_every_key():
    vocab = {'[PAD]': 0, '中': 5, '##ab': 7, 'ab': 9, '\ud800': 11, 'ß': 12}
    t = df.vocab_table(vocab)
    n = len(t['slots'])
    assert n & (n - 1) == 0 and n >= 2 * len(vocab) and t['max_piece'] == 5
    blob = t['blob'].tobytes()
    for key, i in vocab.items():
        data = key.encode('utf-8', 'surrogatepass')
        s = df._fnv1a(data) & (n - 1)
        while True:
            e = t['slots'][s]
            assert e >= 0, key
            off, ln, eid = t['entries'][e]
            if blob[off:off + ln] == data:
                assert eid == i
                break
            s = (s + 1) & (n - 1)
    with pytest.raises(ValueError):
        df.vocab_table({'x': 1 << 24})


def test_featurizer_refuses_other_tokenizers():
    with pytest.raises(TypeError):
        df.DeviceFeaturizer(object(), 16, 'cpu')
    with pytest.raises(TypeError):
        df.DeviceFeaturizer({'[PAD]': 0}, 16, 'cpu')


def _offsets(vals):
    arr = (ctypes.c_int64 * len(vals))(*vals)
    return arr


def test_featurize_abi_rejects_bad_arguments_before_any_cuda_call():
    h = _lib.lib()
    good = _offsets([0, 3, 5])

    def wp(B=2, L=8, offs=good, text=1, n_slots=4, out=1, max_piece=1):
        return h.ner_featurize_wordpiece(text, 1, ctypes.addressof(offs) if offs is not None else None, B, L, 1, 1, 1, 1,
                                         n_slots, 1, 1, max_piece, 1, 1, 2, 0, 3, out, 1, 1, 1, 1, None)

    def ch(B=2, L=8, offs=good, text=1, n_slots=4, out=1):
        return h.ner_featurize_chars(text, 1, ctypes.addressof(offs) if offs is not None else None, B, L, 1, 1, 1,
                                     n_slots, 1, 1, 0, 1, out, 1, 1, 1, 1, None)

    for fn in (wp, ch):
        assert fn(B=-1) == -1
        assert fn(B=0) == 0                       # empty batch: no-op
        assert fn(L=0) == -1
        assert fn(text=None) == -1
        assert fn(out=None) == -1
        assert fn(offs=None) == -1
        assert fn(n_slots=6) == -1                # not a power of two
        assert fn(offs=_offsets([0, 5, 3])) == -1     # not monotone
        assert fn(offs=_offsets([1, 3, 5])) == -1     # does not start at 0
        assert fn(B=1 << 16, L=1 << 15, offs=_offsets([0] * ((1 << 16) + 1))) == -2
    assert wp(L=1) == -1                          # [CLS] and [SEP] need two positions
    assert wp(B=0, L=1) == -1
    assert wp(max_piece=0) == -1
