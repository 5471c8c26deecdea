"""ner_bigru_recurrence and ner_bigru_recurrence_bwd (the GRU cell of the bidirectional RNN layer) reject bad arguments
before any CUDA call, so this runs without a GPU."""
from chinesener_b200 import _lib


def test_bigru_entry_points_are_registered():
    h = _lib.lib()
    for name in ("ner_bigru_recurrence", "ner_bigru_recurrence_bwd"):
        assert name in _lib.SIGNATURES
        assert getattr(h, name).argtypes == _lib.SIGNATURES[name][1]


def test_bigru_recurrence_argument_checks():
    h = _lib.lib()

    def fwd(B=4, L=8, H=128, ld=None, act=0, keep=1.0, ptrs=1, gates=None, hstate=None, rh=None):
        # (xproj, wh_fw, wh_bw, seq_len, out, B, L, H, ld_xproj, activation, cu_seqlens, gates_out, hstate_out, rh_out,
        #  keep_prob, seed, stream)
        p = ptrs or None
        ld = 6 * H if ld is None else ld
        return h.ner_bigru_recurrence(p, p, p, p, p, B, L, H, ld, act, None, gates, hstate, rh, keep, 0, None)

    assert fwd(ptrs=0) == -1                         # null pointers
    assert fwd(B=-1) == -1
    assert fwd(L=0) == -1
    assert fwd(H=0) == -1
    assert fwd(H=100, ld=599) == -1                  # xproj row stride below 6H
    assert fwd(act=2) == -1                          # activation: 0 tanh, 1 relu
    assert fwd(keep=0.0) == -1
    assert fwd(keep=1.5) == -1
    assert fwd(gates=1) == -1                        # training saves: all three or none
    assert fwd(gates=1, hstate=1) == -1
    assert fwd(hstate=1, rh=1) == -1
    assert fwd(H=102) == -2                          # H % 4 != 0
    assert fwd(H=512) == -2                          # recurrent slice does not fit an 8-CTA cluster
    assert fwd(B=0, ptrs=0) == 0                     # empty batch: no-op


def test_bigru_recurrence_bwd_argument_checks():
    h = _lib.lib()

    def bwd(B=4, L=8, H=128, act=0, keep=1.0, ptrs=1, hstate=1):
        # (d_out, gates, hstate, wh_fw, wh_bw, seq_len, d_xproj, B, L, H, activation, keep_prob, seed, stream)
        p = ptrs or None
        return h.ner_bigru_recurrence_bwd(p, p, hstate or None, p, p, p, p, B, L, H, act, keep, 0, None)

    assert bwd(ptrs=0) == -1
    assert bwd(hstate=0) == -1                       # the carried h is required
    assert bwd(B=-1) == -1
    assert bwd(L=0) == -1
    assert bwd(H=-4) == -1
    assert bwd(act=-1) == -1
    assert bwd(keep=0.0) == -1
    assert bwd(keep=2.0) == -1
    assert bwd(H=130) == -2
    assert bwd(H=1024) == -2
    assert bwd(B=0, ptrs=0, hstate=0) == 0


def test_bad_rnn_settings_raise_before_any_kernel():
    """cell_type outside {'lstm', 'gru'} raises in PREDICT and TRAIN; a hidden_units_list / keep_prob_list shorter than
    cell_size is a ValueError naming the list (the reference fails with an IndexError)."""
    import pytest
    import torch

    from chinesener_b200 import variables
    from chinesener_b200.tools import layer

    x = torch.zeros(2, 5, 8)
    lens = torch.tensor([5, 3], dtype=torch.int32)
    store = variables.VariableStore("cpu")
    with variables.use_store(store):
        for training in (False, True):
            with pytest.raises(Exception, match="cell_type"):
                layer.bilstm(x, "rnn", "tanh", [16], [1.0], 1, lens, "float32", training)
            with pytest.raises(ValueError, match="keep_prob_list"):
                layer.bilstm(x, "gru", "tanh", [16, 16], [1.0], 2, lens, "float32", training)
            with pytest.raises(ValueError, match="hidden_units_list"):
                layer.bilstm(x, "lstm", "tanh", [16], [1.0, 1.0], 2, lens, "float32", training)
    assert not store.vars
