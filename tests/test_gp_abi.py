"""ner_gp_* (the bert_global_pointer kernels) are exported and declared, reject bad arguments before any CUDA call, and the
plugin refuses unsupported settings and document mode with a ValueError before any launch; all without a GPU."""
import os

import pytest

from chinesener_b200 import _lib, windows
from chinesener_b200.data import mrc
from chinesener_b200.model import bert_global_pointer

NAMES = ["ner_gp_targets", "ner_gp_rope", "ner_gp_rope_bwd", "ner_gp_loss_workspace_bytes", "ner_gp_loss_fwd",
         "ner_gp_loss_bwd", "ner_gp_decode_workspace_bytes", "ner_gp_decode"]
Q = 16                     # a non-null, 16-byte aligned fake pointer: never dereferenced when a check fails


def test_registered_and_declared():
    header = open(os.path.join(os.path.dirname(__file__), "..", "include", "ner_b200.h")).read()
    h = _lib.lib()
    for n in NAMES:
        assert n in _lib.SIGNATURES and n + "(" in header
        assert getattr(h, n) is not None


def test_targets_and_rope_argument_checks():
    h = _lib.lib()
    # (label_ids, seq_len, type_tag, B, T, L, span_end, stream)
    assert h.ner_gp_targets(Q, Q, Q, 2, 3, 8, None, None) == -1
    assert h.ner_gp_targets(Q, Q, Q, -1, 3, 8, Q, None) == -1
    assert h.ner_gp_targets(Q, Q, Q, 2, 0, 8, Q, None) == -1
    assert h.ner_gp_targets(Q, Q, Q, 2, 33, 8, Q, None) == -2
    assert h.ner_gp_targets(Q, Q, Q, 2, 3, 513, Q, None) == -2
    assert h.ner_gp_targets(Q, Q, Q, 4096, 32, 512, Q, None) == -2            # B*T*L*L >= 2^31
    assert h.ner_gp_targets(None, None, None, 0, 3, 8, None, None) == 0       # B = 0: no-op
    # (proj, ld, cu, B, T, L, hi, lo, stream)
    assert h.ner_gp_rope(Q, 380, None, 2, 3, 8, Q, None, None) == -1          # ld < T*2D
    assert h.ner_gp_rope(Q, 385, None, 2, 3, 8, Q, None, None) == -1          # odd ld
    assert h.ner_gp_rope(None, 384, None, 2, 3, 8, Q, None, None) == -1
    assert h.ner_gp_rope(Q, 384, None, 2, 3, 8, 24, None, None) == -1         # rot_hi not 16-byte aligned
    assert h.ner_gp_rope(Q, 128 * 33, None, 2, 33, 8, Q, None, None) == -2
    assert h.ner_gp_rope(Q, 384, None, 2, 3, 600, Q, None, None) == -2
    # (d_rot, cu, B, T, L, d_proj, ld, stream)
    assert h.ner_gp_rope_bwd(Q, None, 2, 3, 8, None, 384, None) == -1
    assert h.ner_gp_rope_bwd(Q, None, 2, 3, 8, Q, 256, None) == -1
    assert h.ner_gp_rope_bwd(Q, None, 2, 3, 513, Q, 384, None) == -2


def test_loss_argument_checks():
    h = _lib.lib()

    def fwd(B=2, T=3, L=8, hi=Q, lo=None, end=Q, loss=Q, ws=Q, nbytes=1 << 20):
        # (hi, lo, seq_len, cu, span_end, B, T, L, loss, lse, workspace, bytes, stream)
        return h.ner_gp_loss_fwd(hi, lo, Q, None, end, B, T, L, loss, Q, ws, nbytes, None)
    assert fwd(hi=None) == -1 and fwd(end=None) == -1 and fwd(loss=None) == -1
    assert fwd(hi=24) == -1 and fwd(lo=40) == -1                               # operands not 16-byte aligned
    assert fwd(T=33) == -2 and fwd(L=513) == -2 and fwd(T=0) == -1
    assert fwd(ws=None) == -3 and fwd(nbytes=16) == -3                         # missing / short workspace
    assert fwd(B=0, hi=None, end=None, loss=None, ws=None) == 0
    assert h.ner_gp_loss_workspace_bytes(2, 3, 130) == 2 * 3 * 3 * 16
    assert h.ner_gp_loss_workspace_bytes(2, 33, 130) == 0

    # (rot, seq_len, cu, span_end, lse, B, T, L, d_loss, d_rot, stream)
    assert h.ner_gp_loss_bwd(Q, Q, None, Q, None, 2, 3, 8, 1.0, Q, None) == -1
    assert h.ner_gp_loss_bwd(Q, Q, None, Q, Q, 2, 3, 8, 1.0, 24, None) == -1
    assert h.ner_gp_loss_bwd(Q, Q, None, Q, Q, 2, 40, 8, 1.0, Q, None) == -2
    assert h.ner_gp_loss_bwd(None, None, None, None, None, 0, 3, 8, 1.0, None, None) == 0


def test_decode_argument_checks():
    h = _lib.lib()

    def dec(B=2, T=3, L=8, cap=8, hi=Q, spans=Q, ws=Q, nbytes=1 << 20):
        # (hi, lo, seq_len, cu, type_tag, B, T, L, o, cls, sep, cap, pred, spans, probs, counts, ws, bytes, stream)
        return h.ner_gp_decode(hi, None, Q, None, Q, B, T, L, 1, 8, 9, cap, Q, spans, Q, Q, ws, nbytes, None)
    assert dec(hi=None) == -1 and dec(cap=-1) == -1 and dec(B=-1) == -1
    assert dec(spans=None) == -1                                               # spans needed when cap > 0
    assert dec(spans=None, cap=0, ws=None) == -3
    assert dec(T=33) == -2 and dec(L=513) == -2
    assert dec(ws=None) == -3 and dec(nbytes=2 * 3 * 64 * 4 - 1) == -3
    assert dec(B=0, hi=None, spans=None, ws=None) == 0
    assert h.ner_gp_decode_workspace_bytes(2, 3, 8) == 2 * 3 * 64 * 4


def _tags(T):
    idx2tag = {0: '[PAD]', 1: 'O'}
    for t in range(T):
        idx2tag[2 + 2 * t], idx2tag[3 + 2 * t] = f'B-T{t}', f'I-T{t}'
    return idx2tag


def test_plugin_refuses_unsupported_settings():
    p = dict(bert_global_pointer.TRAIN_PARAMS)
    assert p['diff_lr_times'] == {'logit': 500}
    assert 'logit' in bert_global_pointer.SCOPE and bert_global_pointer.HEAD == 64
    ok = mrc.TypeTable(dict(p, idx2tag=_tags(3), max_seq_len=512), device='cpu')
    bert_global_pointer.check_supported(p, ok)
    assert ok.names == ['T0', 'T1', 'T2'] and ok.type_tag.tolist() == [[2, 3], [4, 5], [6, 7]]
    assert (ok.o_tag, ok.cls_tag, ok.sep_tag) == (1, 1, 1)
    with pytest.raises(ValueError, match="512"):
        bert_global_pointer.check_supported(p, mrc.TypeTable(dict(p, idx2tag=_tags(3), max_seq_len=513), device='cpu'))
    with pytest.raises(ValueError):
        mrc.TypeTable(dict(p, idx2tag=_tags(33), max_seq_len=128), device='cpu')           # T > 32
    with pytest.raises(ValueError):
        mrc.TypeTable(dict(p, idx2tag={0: 'O', 1: '[CLS]'}, max_seq_len=128), device='cpu')  # no entity type
    with pytest.raises(ValueError):
        mrc.TypeTable(dict(p, idx2tag={0: '[PAD]', 1: 'B-X', 2: 'I-X'}, max_seq_len=128), device='cpu')   # no 'O'


def test_document_mode_is_refused():
    windows.check_batch('bert_global_pointer', 128, 512)
    with pytest.raises(ValueError, match=r"\[B, T, L, L\]"):
        windows.check_batch('bert_global_pointer', 600, 512)
