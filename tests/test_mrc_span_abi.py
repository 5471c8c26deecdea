"""ner_mrc_span_* (the bert_mrc_span kernels) reject bad arguments before any CUDA call, are registered in _lib, and the
plugin refuses unsupported settings and document mode with a ValueError before any launch; all without a GPU."""
import pytest

from chinesener_b200 import _lib, windows
from chinesener_b200.data import mrc
from chinesener_b200.model import bert_mrc_span

NAMES = ["ner_mrc_span_targets", "ner_mrc_span_match_fwd_workspace_bytes", "ner_mrc_span_match_fwd",
         "ner_mrc_span_match_bwd_workspace_bytes", "ner_mrc_span_match_bwd", "ner_mrc_span_decode_workspace_bytes",
         "ner_mrc_span_decode"]


def test_registered_and_declared():
    import os
    header = open(os.path.join(os.path.dirname(__file__), "..", "include", "ner_b200.h")).read()
    h = _lib.lib()
    for n in NAMES:
        assert n in _lib.SIGNATURES and n + "(" in header
        assert getattr(h, n) is not None


def test_targets_argument_checks():
    h = _lib.lib()
    # (pair_labels, pair_seq_len, P, L, start_y, end_y, span_end, stream)
    assert h.ner_mrc_span_targets(None, None, 4, 8, None, None, None, None) == -1
    assert h.ner_mrc_span_targets(16, 16, 4, 8, 16, 16, None, None) == -1
    assert h.ner_mrc_span_targets(16, 16, -1, 8, 16, 16, 16, None) == -1
    assert h.ner_mrc_span_targets(16, 16, 4, 0, 16, 16, 16, None) == -1
    assert h.ner_mrc_span_targets(16, 16, 4, 512, 16, 16, 16, None) == -2       # longer than the pair bound
    assert h.ner_mrc_span_targets(None, None, 0, 8, None, None, None, None) == 0  # empty: no-op


def _fwd(P=4, L=8, I=64, ld=128, keep=1.0, ptrs=16, end=16, loss=16, ws=16, nbytes=1 << 20):
    # (uv, ld, b1, w2, b2, seq_len, span_end, P, L, I, keep, seed, z, loss, workspace, bytes, stream)
    q = ptrs or None
    return _lib.lib().ner_mrc_span_match_fwd(q, ld, q, q, q, q, end or None, P, L, I, keep, 7, q, loss or None, ws or None,
                                             nbytes, None)


def test_match_fwd_argument_checks():
    assert _fwd(ptrs=0) == -1
    assert _fwd(P=-1) == -1
    assert _fwd(L=0) == -1
    assert _fwd(L=512) == -2
    assert _fwd(I=48, ld=96) == -2                  # I % 32 != 0
    assert _fwd(I=4128, ld=8256) == -2               # I > 4096
    assert _fwd(ld=100) == -1                        # ld < 2I
    assert _fwd(ld=130) == -1                        # ld % 4 != 0
    assert _fwd(keep=0.0) == -1 and _fwd(keep=1.5) == -1
    assert _fwd(end=0) == -1                         # a loss needs the targets
    assert _fwd(ws=0) == -3 and _fwd(nbytes=4) == -3
    assert _fwd(ptrs=17) == -1                       # uv not 16-byte aligned
    assert _fwd(P=0, ptrs=0, end=0, loss=0, ws=0) == 0
    assert _lib.lib().ner_mrc_span_match_fwd_workspace_bytes(4, 40) == 4 * 4 * 2 * 2


def test_match_bwd_argument_checks():
    h = _lib.lib()

    def bwd(P=4, L=8, I=64, ld=128, keep=0.9, ptrs=16, d_b2=16, ws=16, nbytes=1 << 20):
        # (uv, ld, z, b1, w2, seq_len, span_end, P, L, I, d_loss, keep, seed, d_uv, d_b1, d_w2, d_b2, ws, bytes, stream)
        q = ptrs or None
        return h.ner_mrc_span_match_bwd(q, ld, q, q, q, q, q, P, L, I, 1.0, keep, 7, q, q, q, d_b2 or None, ws or None,
                                        nbytes, None)
    assert bwd(ptrs=0) == -1
    assert bwd(d_b2=0) == -1
    assert bwd(L=600) == -2 and bwd(I=40, ld=80) == -2
    assert bwd(keep=-0.1) == -1
    assert bwd(ws=0) == -3 and bwd(nbytes=8) == -3
    assert bwd(P=0, ptrs=0, d_b2=0, ws=0) == 0
    assert h.ner_mrc_span_match_bwd_workspace_bytes(3, 64) == (2 * 3 * 64 + 3) * 4


def test_decode_argument_checks():
    h = _lib.lib()

    def dec(B=2, T=3, L=8, I=64, ld=128, cap=8, ptrs=16, spans=16, ws=16, nbytes=1 << 20):
        # (start, end, uv, ld, b1, w2, b2, seq_len, type_tag, B, T, L, I, o, cls, sep, cap, pred, spans, probs, counts, ws,
        #  bytes, stream)
        q = ptrs or None
        return h.ner_mrc_span_decode(q, q, q, ld, q, q, q, q, q, B, T, L, I, 1, 8, 9, cap, q, spans or None, q, q, ws or None,
                                     nbytes, None)
    assert dec(ptrs=0) == -1
    assert dec(B=-1) == -1 and dec(T=0) == -1 and dec(cap=-1) == -1
    assert dec(T=33) == -2
    assert dec(L=512) == -2 and dec(I=96 + 16, ld=224) == -2
    assert dec(spans=0) == -1                        # spans needed when cap > 0
    assert dec(ws=0) == -3 and dec(nbytes=100) == -3
    assert dec(B=0, ptrs=0, spans=0, ws=0) == 0
    assert h.ner_mrc_span_decode_workspace_bytes(6, 8) == (6 * 64 + 6 * 16 + 12) * 4


class _Table:
    def __init__(self, L):
        self.L = L


def test_plugin_refuses_unsupported_settings():
    base = dict(bert_mrc_span.TRAIN_PARAMS)
    assert base['mrc_span_hidden'] == 1024 and base['mrc_dropout'] == 0.1
    assert base['diff_lr_times'] == {'logit': 500}
    assert bert_mrc_span.check_supported(base, _Table(128)) == (1024, 0.9)
    for bad in ({'mrc_span_hidden': 1000}, {'mrc_span_hidden': 8192}, {'mrc_span_hidden': 0}, {'mrc_dropout': 1.0},
                {'mrc_dropout': -0.5}):
        with pytest.raises(ValueError):
            bert_mrc_span.check_supported(dict(base, **bad), _Table(128))
    with pytest.raises(ValueError, match="511"):
        bert_mrc_span.check_supported(base, _Table(512))
    many = {0: 'O'}
    for t in range(33):
        many[1 + 2 * t], many[2 + 2 * t] = f'B-T{t}', f'I-T{t}'
    with pytest.raises(ValueError):
        mrc.entity_types(many)


def test_document_mode_is_refused():
    assert windows.REFUSED['bert_mrc_span'] == windows.REFUSED['bert_mrc']
    windows.check_batch('bert_mrc_span', 128, 512)
    with pytest.raises(ValueError, match="query repeated"):
        windows.check_batch('bert_mrc_span', 600, 512)
