"""Token-level losses with the reference's function surface (reference tools/loss.py), over the softmax-head kernels
`ner_token_xent` and `ner_token_dice` (csrc/token_head.cu).

`cross_entropy_loss` is the loss of the `bert_ce` plugin, `dice_loss` that of `bert_dice`.  The reference file is not
part of this repository (SURVEY.md §2.1 records it as "masked CE, dice"), so both are restatements, not pinned parity
points: the loss of every token with t < seq_len, averaged over those tokens (tf.boolean_mask + tf.reduce_mean), 0 for a
batch without tokens.  A different reduction only rescales the gradient; pred_ids, and so F1, do not depend on it.
`dice_loss` is the self-adjusting Dice loss of Li et al., "Dice Loss for Data-imbalanced NLP Tasks" (ACL 2020), summed
over the classes of a token (formula in include/ner_b200.h, ner_token_dice).
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


def dice_loss(logits, labels, seq_len, max_seq_len, alpha, gamma, is_training):
    """mean over t < seq_len of the self-adjusting Dice loss of softmax(logits) (sum over the K classes, (1-p)^alpha
    weighting, smoothing gamma), logits [B, L, K<=32] f32 with L = max_seq_len.  -> scalar loss; None without labels.

    TRAIN: ONE kernel launch computes the loss, d loss / d logits and the argmax; the tape entry hands d_logits to
    `logits`, and the argmax rides along as `loss.pred_ids` [B, L] int32.
    EVAL / PREDICT: a `variables.Deferred`, evaluated only when the loss is fetched (never in PREDICT)."""
    if labels is None:
        return None
    assert logits.shape[1] == max_seq_len, (tuple(logits.shape), max_seq_len)
    tape = autodiff.current() if is_training else None
    lg = logits.contiguous()
    if tape is None:
        return variables.Deferred(lambda: ops.token_dice(lg, labels, seq_len, alpha, gamma, want_pred=False)[1])
    pred, loss, d_logits = ops.token_dice(lg, labels, seq_len, alpha, gamma, want_grad=True, d_loss=1.0)
    loss.pred_ids = pred
    tape.record(loss, lambda g: tape.add_grad(logits, d_logits))
    return loss


def argmax(logits):
    """tf.argmax(logits, axis=-1) as int32 [B, L]: the first maximum at EVERY position (no zero fill past seq_len)."""
    return ops.token_xent(logits.contiguous(), want_pred=True)[0]
