"""ner_token_xent (the bert_ce softmax head) rejects bad arguments before any CUDA call, so this runs without a GPU."""
from chinesener_b200 import _lib


def test_token_xent_argument_checks():
    h = _lib.lib()
    assert h.ner_token_xent_scratch_floats() >= 16 + 8
    # (logits, labels, seq_len, pred_ids, loss, d_logits, d_loss, scratch, B, L, K, stream)
    assert h.ner_token_xent(None, None, None, None, None, None, 1.0, None, 4, 8, 10, None) == -1     # null logits
    assert h.ner_token_xent(1, None, None, 1, None, None, 1.0, None, -1, 8, 10, None) == -1          # negative B
    assert h.ner_token_xent(1, None, None, 1, None, None, 1.0, None, 4, 0, 10, None) == -1           # L = 0
    assert h.ner_token_xent(1, None, None, 1, None, None, 1.0, None, 4, 8, 0, None) == -1            # K = 0
    assert h.ner_token_xent(1, None, None, 1, None, None, 1.0, None, 4, 8, 33, None) == -2           # K > 32
    assert h.ner_token_xent(None, None, None, None, None, None, 1.0, None, 0, 8, 10, None) == 0      # empty batch: no-op
    assert h.ner_token_xent(1, None, None, 1, 1, None, 1.0, None, 4, 8, 10, None) == -1              # loss needs labels
    assert h.ner_token_xent(1, 1, None, 1, 1, None, 1.0, 1, 4, 8, 10, None) == -1                    # labels need seq_len
    assert h.ner_token_xent(1, 1, 1, 1, 1, None, 1.0, None, 4, 8, 10, None) == -1                    # ... and scratch
