"""CPU: ner_augment_rows / ner_vocab_sample are declared, exported and bound, and reject bad arguments before any CUDA
call."""
import os
import re

from chinesener_b200 import _lib

INVALID, UNSUPPORTED = -1, -2
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P16 = 1 << 20          # a 16-byte aligned fake pointer: no argument check dereferences it


def _rows(B=2, L=8, K=10, T=3, probs=(0.5, 0.3, 0.3, 0.3, 0.0), sizes=(4, 9, 30), mask_id=103, mlm=False, null=None):
    p = [P16] * 19      # 5 inputs, tag_class, type_tag, 3 mention arrays, 2 tag arrays, 5 outputs, mlm_ids, mlm_positions
    if not mlm:
        p[17] = p[18] = None
    if null is not None:
        p[null] = None
    n_men, n_men_tok, n_tag_tok = sizes
    return _lib.lib().ner_augment_rows(*p[:5], B, L, p[5], K, p[6], T, p[7], p[8], p[9], n_men, n_men_tok, p[10], p[11],
                                       n_tag_tok, *probs, 7, 0, 0, mask_id, *p[12:19], None)


def _sample(M=4, V=100, ld=100, T=1.0, logits=P16, null=None):
    p = [P16] * 3       # eligible, positions, token_ids
    if null is not None:
        p[null] = None
    return _lib.lib().ner_vocab_sample(logits, ld, V, p[0], p[1], M, 1000, T, 7, p[2], None)


def test_symbols_are_declared_exported_and_bound():
    with open(os.path.join(ROOT, "include", "ner_b200.h")) as f:
        header = f.read()
    for name in ("ner_augment_rows", "ner_augment_rows_smem_bytes", "ner_vocab_sample"):
        assert re.search(r"\b%s\(" % name, header), name
        assert name in _lib.SIGNATURES
        assert getattr(_lib.lib(), name) is not None
    smem = _lib.lib().ner_augment_rows_smem_bytes
    assert smem(128) == 16 * 128 + 8 * 128
    assert smem(4095) == 16 * 4095 + 8 * 4096 and smem(127) == 16 * 127 + 8 * 128
    assert smem(0) == 0 and smem(4096) == 0


def test_rows_argument_checks():
    assert _rows(B=-1) == INVALID
    assert _rows(L=0) == INVALID
    assert _rows(K=0) == INVALID
    assert _rows(T=-1) == INVALID
    assert _rows(L=4096) == UNSUPPORTED
    assert _rows(K=129) == UNSUPPORTED
    assert _rows(B=1 << 20, L=4095) == UNSUPPORTED                     # B * L >= 2^31
    for i in range(5):
        for bad in (-0.1, 1.5, float("nan")):
            probs = [0.5, 0.3, 0.3, 0.3, 0.0]
            probs[i] = bad
            assert _rows(probs=tuple(probs), mlm=True) == INVALID, (i, bad)
    assert _rows(sizes=(-1, 9, 30)) == INVALID
    assert _rows(sizes=(4, -1, 30)) == INVALID
    assert _rows(sizes=(4, 9, -1)) == INVALID
    assert _rows(probs=(0.5, 0, 0, 0, 0.2)) == INVALID                  # mlm without its outputs
    assert _rows(probs=(0.5, 0, 0, 0, 0.2), mlm=True, mask_id=-1) == INVALID
    assert _rows(mlm=True, null=18) == INVALID                          # only one of mlm_ids / mlm_positions
    assert _rows(B=0, null=0) == 0                                      # empty batch: no-op
    for i in list(range(6)) + list(range(12, 17)):                      # always read
        assert _rows(null=i) == INVALID, i
    for i in (6, 7, 8, 9):                                              # read by mr only
        assert _rows(null=i) == INVALID, i
        assert _rows(null=i, probs=(0.5, 0, 0.3, 0.3, 0), B=0) == 0, i
    for i in (10, 11):                                                  # read by lwtr only
        assert _rows(null=i) == INVALID, i
    assert _rows(T=0) == INVALID                                        # mr needs a type


def test_sample_argument_checks():
    assert _sample(M=-1) == INVALID
    assert _sample(V=0) == INVALID
    assert _sample(V=100, ld=96) == INVALID
    assert _sample(V=99, ld=99) == INVALID
    assert _sample(V=50001, ld=50004) == UNSUPPORTED
    for T in (0.0, -1.0, float("inf"), float("nan")):
        assert _sample(T=T) == INVALID, T
    assert _sample(logits=P16 + 4) == INVALID
    assert _sample(logits=None) == INVALID
    for i in range(3):
        assert _sample(null=i) == INVALID, i
    assert _sample(M=0, logits=None, null=0) == 0
