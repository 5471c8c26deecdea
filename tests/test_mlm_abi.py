"""CPU: ner_mlm_mask / ner_vocab_xent are exported and declared and reject bad arguments before any CUDA call."""
import os
import re

from chinesener_b200 import _lib

INVALID, UNSUPPORTED = -1, -2
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("ner_mlm_mask", "ner_vocab_xent")
P16 = 1 << 20          # a 16-byte aligned fake pointer: no argument check dereferences it


def _mask(B=2, L=8, V=100, mask_id=3, ptrs=None):
    p = [P16] * 7 if ptrs is None else ptrs     # token_ids, seq_len, word_start, pred_offsets, masked_ids, positions, labels
    return _lib.lib().ner_mlm_mask(*p[:4], B, L, 7, V, mask_id, *p[4:], None)


def _xent(M=4, V=100, ld=100, ptrs=None, logits=P16, d_logits=P16):
    p = [P16] * 6 if ptrs is None else ptrs     # labels, loss, count, correct, pred, scratch
    return _lib.lib().ner_vocab_xent(logits, ld, p[0], M, V, 1.0, p[1], p[2], p[3], p[4], d_logits, p[5], None)


def test_symbols_are_declared_exported_and_bound():
    with open(os.path.join(ROOT, "include", "ner_b200.h")) as f:
        header = f.read()
    for name in NAMES + ("ner_vocab_xent_scratch_floats",):
        assert re.search(r"\b%s\(" % name, header), name
        assert name in _lib.SIGNATURES
        assert getattr(_lib.lib(), name) is not None
    assert _lib.lib().ner_vocab_xent_scratch_floats(100) >= 200


def test_mask_argument_checks():
    assert _mask(B=-1) == INVALID
    assert _mask(L=0) == INVALID
    assert _mask(L=513) == UNSUPPORTED
    assert _mask(V=0) == INVALID
    assert _mask(V=50001, mask_id=3) == UNSUPPORTED
    assert _mask(mask_id=-1) == INVALID
    assert _mask(V=100, mask_id=100) == INVALID
    assert _mask(B=1 << 22, L=512) == UNSUPPORTED                # B * L >= 2^31
    assert _mask(B=0, ptrs=[None] * 7) == 0                        # empty batch: no-op
    for i in range(7):
        if i == 2:                                                 # word_start is optional
            continue
        p = [P16] * 7
        p[i] = None
        assert _mask(ptrs=p) == INVALID, i


def test_xent_argument_checks():
    assert _xent(M=-1) == INVALID
    assert _xent(V=0) == INVALID
    assert _xent(V=50001, ld=50004) == UNSUPPORTED
    assert _xent(V=100, ld=96) == INVALID                          # ld < V
    assert _xent(V=99, ld=99) == INVALID                           # ld % 4
    assert _xent(logits=P16 + 4) == INVALID                        # logits not 16-byte aligned
    assert _xent(d_logits=P16 + 2) == INVALID                      # d_logits not 8-byte aligned
    assert _xent(M=0, ptrs=[None] * 6, logits=None, d_logits=None) == 0     # no rows: no-op
    assert _xent(logits=None) == INVALID
    for i in range(6):
        if i == 4:                                                 # pred is optional
            continue
        p = [P16] * 6
        p[i] = None
        assert _xent(ptrs=p) == INVALID, i
