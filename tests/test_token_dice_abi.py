"""ner_token_dice (the bert_dice softmax head) rejects bad arguments before any CUDA call, so this runs without a GPU."""
from chinesener_b200 import _lib


def test_token_dice_argument_checks():
    h = _lib.lib()
    f = h.ner_token_dice
    # (logits, labels, seq_len, pred_ids, loss, d_logits, d_loss, alpha, gamma, scratch, B, L, K, stream)
    assert f(None, 1, 1, 1, 1, None, 1.0, 1.0, 1.0, 1, 4, 8, 10, None) == -1                     # null logits
    assert f(1, 1, 1, 1, 1, None, 1.0, 1.0, 1.0, 1, -1, 8, 10, None) == -1                       # negative B
    assert f(1, 1, 1, 1, 1, None, 1.0, 1.0, 1.0, 1, 4, 0, 10, None) == -1                        # L = 0
    assert f(1, 1, 1, 1, 1, None, 1.0, 1.0, 1.0, 1, 4, 8, 0, None) == -1                         # K = 0
    assert f(1, 1, 1, 1, 1, None, 1.0, 1.0, 1.0, 1, 4, 8, 33, None) == -2                        # K > 32
    assert f(1, 1, 1, 1, 1, None, 1.0, 1.0, 1.0, 1, 1 << 20, 1 << 12, 10, None) == -2            # B * L >= 2^31
    assert f(None, None, None, None, None, None, 1.0, 1.0, 1.0, None, 0, 8, 10, None) == 0       # empty batch: no-op
    assert f(1, None, 1, 1, None, None, 1.0, 1.0, 1.0, 1, 4, 8, 10, None) == -1                  # labels are required
    assert f(1, 1, None, 1, 1, None, 1.0, 1.0, 1.0, 1, 4, 8, 10, None) == -1                     # ... and seq_len
    assert f(1, 1, 1, 1, 1, None, 1.0, 1.0, 1.0, None, 4, 8, 10, None) == -1                     # ... and scratch
    for alpha, gamma in ((-1.0, 1.0), (-1e-30, 1.0), (float('nan'), 1.0), (float('inf'), 1.0),
                         (1.0, 0.0), (1.0, -0.5), (1.0, float('nan')), (1.0, float('inf'))):
        assert f(1, 1, 1, 1, 1, None, 1.0, alpha, gamma, 1, 4, 8, 10, None) == -1, (alpha, gamma)
    assert f(1, 1, 1, None, None, None, 1.0, 0.0, 1e-3, 1, 4, 8, 10, None) == 0                  # valid, nothing to write
