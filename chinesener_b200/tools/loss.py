"""Token-level losses with the reference's function surface (reference tools/loss.py), over the softmax-head kernel
`ner_token_xent` (csrc/token_head.cu).

`cross_entropy_loss` is the loss of the `bert_ce` plugin.  The reference file is not part of this repository (SURVEY.md
§2.1 records it as "masked CE, dice"), so the reduction below is a restatement, not a pinned parity point: the cross
entropy of every token with t < seq_len, averaged over those tokens (tf.boolean_mask + tf.reduce_mean), 0 for a batch
without tokens.  A different reduction only rescales the gradient; pred_ids, and so F1, do not depend on it.
"""
from .. import autodiff, ops, variables


def cross_entropy_loss(logits, labels, seq_len, max_seq_len, is_training):
    """mean over t < seq_len of sparse_softmax_cross_entropy(labels, logits), logits [B, L, K<=32] f32 with
    L = max_seq_len.  -> scalar loss; None without labels.

    TRAIN: ONE kernel launch computes the loss, d loss / d logits and the argmax; the tape entry hands d_logits to
    `logits`, and the argmax rides along as `loss.pred_ids` [B, L] int32.
    EVAL / PREDICT: a `variables.Deferred`, evaluated only when the loss is fetched (never in PREDICT)."""
    if labels is None:
        return None
    assert logits.shape[1] == max_seq_len, (tuple(logits.shape), max_seq_len)
    tape = autodiff.current() if is_training else None
    lg = logits.contiguous()
    if tape is None:
        return variables.Deferred(lambda: ops.token_xent(lg, labels, seq_len, want_pred=False)[1])
    pred, loss, d_logits = ops.token_xent(lg, labels, seq_len, want_grad=True, d_loss=1.0)
    loss.pred_ids = pred
    tape.record(loss, lambda g: tape.add_grad(logits, d_logits))
    return loss


def argmax(logits):
    """tf.argmax(logits, axis=-1) as int32 [B, L]: the first maximum at EVERY position (no zero fill past seq_len)."""
    return ops.token_xent(logits.contiguous(), want_pred=True)[0]
