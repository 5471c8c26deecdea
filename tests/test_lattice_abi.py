"""ner_lattice_recurrence / ner_lattice_recurrence_bwd / ner_lexicon_build_lattice reject bad arguments before any CUDA
call, so this runs without a GPU."""
from chinesener_b200 import _lib

INVALID, UNSUPPORTED = -1, -2


def _fwd(B=2, L=8, H=16, Kw=4, ptrs=None, saves=None):
    p = [1] * 9 if ptrs is None else ptrs
    s = [None] * 7 if saves is None else saves
    return _lib.lib().ner_lattice_recurrence(*p, B, L, H, Kw, *s, None)


def _bwd(B=2, L=8, H=16, Kw=4, ptrs=None):
    p = [1] * 16 if ptrs is None else ptrs
    return _lib.lib().ner_lattice_recurrence_bwd(*p, B, L, H, Kw, None)


def test_forward_shape_checks():
    assert _fwd(B=-1) == INVALID
    assert _fwd(L=0) == INVALID
    assert _fwd(H=0) == INVALID
    assert _fwd(Kw=0) == INVALID
    assert _fwd(Kw=9) == UNSUPPORTED                      # more word slots than the kernels list
    assert _fwd(H=1024) == UNSUPPORTED                    # recurrent weights do not fit a cluster of 8 CTAs
    assert _fwd(B=0, ptrs=[None] * 9) == 0                # empty batch: no-op


def test_forward_pointer_checks():
    for i in range(9):
        p = [1] * 9
        p[i] = None
        assert _fwd(ptrs=p) == INVALID, i
    for i in range(7):                                    # the saved tensors come all or none
        s = [1] * 7
        s[i] = None
        assert _fwd(saves=s) == INVALID, i


def test_backward_checks():
    assert _bwd(B=-1) == INVALID
    assert _bwd(L=0) == INVALID
    assert _bwd(Kw=0) == INVALID
    assert _bwd(Kw=9) == UNSUPPORTED
    assert _bwd(H=1024) == UNSUPPORTED
    assert _bwd(B=0, ptrs=[None] * 16) == 0
    for i in range(16):
        p = [1] * 16
        p[i] = None
        assert _bwd(ptrs=p) == INVALID, i


def test_lattice_builder_checks():
    f = _lib.lib().ner_lexicon_build_lattice
    # (lexicon, codepoints, sent_offsets, n_sent, max_seq_len, Kw, ids_out, lens_out, dropped_out, n_threads)
    assert f(None, 1, 1, 1, 8, 4, 1, 1, None, 1) == INVALID       # null lexicon
    assert f(1, 1, None, 1, 8, 4, 1, 1, None, 1) == INVALID       # null offsets
    assert f(1, 1, 1, -1, 8, 4, 1, 1, None, 1) == INVALID         # negative count
    assert f(1, 1, 1, 1, 0, 4, 1, 1, None, 1) == INVALID          # max_seq_len 0
    assert f(1, 1, 1, 1, 8, 0, 1, 1, None, 1) == INVALID          # Kw 0
    assert f(1, 1, 1, 1, 8, 9, 1, 1, None, 1) == INVALID          # Kw > 8
    assert f(1, 1, 1, 1, 8, 4, None, 1, None, 1) == INVALID       # null ids
    assert f(1, 1, 1, 1, 8, 4, 1, None, None, 1) == INVALID       # null lens
