"""ner_multihot_embed_fwd / ner_small_table_grad reject bad arguments before any CUDA call, so this runs without a GPU."""
from chinesener_b200 import _lib


def test_multihot_embed_argument_checks():
    f = _lib.lib().ner_multihot_embed_fwd
    # (table, weights, out, n_tok, V, E, ld_out, stream)
    assert f(1, 1, 1, -1, 5, 5, 5, None) == -1                   # negative n_tok
    assert f(1, 1, 1, 4, 0, 5, 5, None) == -1                    # V = 0
    assert f(1, 1, 1, 4, 5, 0, 5, None) == -1                    # E = 0
    assert f(1, 1, 1, 4, 5, 5, 4, None) == -1                    # ld_out < E
    assert f(1, 1, 1, 4, 9, 5, 5, None) == -2                    # V > 8
    assert f(1, 1, 1, 4, 5, 129, 129, None) == -2                # E > 128
    assert f(None, 1, 1, 4, 5, 5, 5, None) == -1                 # null table
    assert f(1, None, 1, 4, 5, 5, 5, None) == -1                 # null weights
    assert f(1, 1, None, 4, 5, 5, 5, None) == -1                 # null out
    assert f(None, None, None, 0, 5, 5, 5, None) == 0            # empty: no-op


def test_small_table_grad_argument_checks():
    h = _lib.lib()
    f = h.ner_small_table_grad
    # (d_table, ids, weights, d_out, n_tok, V, E, ld_dout, scratch, stream)
    assert f(1, 1, None, 1, -1, 5, 5, 5, 1, None) == -1          # negative n_tok
    assert f(1, 1, None, 1, 4, 0, 5, 5, 1, None) == -1           # V = 0
    assert f(1, 1, None, 1, 4, 5, 0, 5, 1, None) == -1           # E = 0
    assert f(1, 1, None, 1, 4, 5, 5, 4, 1, None) == -1           # ld_dout < E
    assert f(1, 1, None, 1, 4, 9, 5, 5, 1, None) == -2           # V > 8
    assert f(1, 1, None, 1, 4, 5, 129, 129, 1, None) == -2       # E > 128
    assert f(1, 1, 1, 1, 4, 5, 5, 5, 1, None) == -1              # ids and weights both given
    assert f(None, 1, 1, None, 0, 5, 5, 5, None, None) == -1     # ... even for an empty batch
    assert f(1, None, None, 1, 4, 5, 5, 5, 1, None) == -1        # neither given
    assert f(None, 1, None, 1, 4, 5, 5, 5, 1, None) == -1        # null d_table
    assert f(1, None, 1, None, 4, 5, 5, 5, 1, None) == -1        # null d_out
    assert f(1, 1, None, 1, 4, 5, 5, 5, None, None) == -1        # null scratch
    assert f(None, None, None, None, 0, 5, 5, 5, None, None) == 0   # empty: no-op
    s = h.ner_small_table_grad_scratch_floats
    assert s(5, 5) > 0 and s(5, 5) % 25 == 0 and s(8, 128) == s(5, 5) // 25 * 1024
    assert s(0, 5) == s(5, 0) == s(9, 5) == s(5, 129) == 0
