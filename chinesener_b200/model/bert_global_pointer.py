"""`bert_global_pointer`: nested NER with the GlobalPointer head (Su, 2021; the head of bert4keras' GlobalPointer) on one
BertModel pass over the plain sentence.  The reference has no GlobalPointer: this is a restatement, parity unpinned.

The types are mrc.entity_types(idx2tag) (every X with a B-X tag, ascending tag id; 1 <= T <= 32) and the head size is
D = 64.  One dense layer global_pointer_logits ([H, T*2D] kernel, [T*2D] bias) gives q and k of every type (bert4keras
layout: q of type t in columns [t*2D, t*2D + D), k after it); both are rotated by RoPE at the token's position in its
padded sentence, and span (i, j) of type t scores s = q'_i . k'_j / sqrt(D) for 1 <= i <= j <= seq_len - 2.  The loss is
bert4keras' global_pointer_crossentropy: per (sentence, type) log(1 + sum_neg e^s) + log(1 + sum_pos e^-s), averaged over
B*T, with the gold spans from the BIO labels (a B-X_t and the I-X_t run after it).  Everything after the projection GEMM
is csrc/global_pointer.cu.

pred_ids [B, L] is in the dataset's tag space: the greedy non-overlapping projection of the spans with s > 0 (the rule of
bert_mrc_span).  The spans themselves ride along as pred_ids.spans [B, cap] (ner_extract_spans' word), pred_ids.span_probs
[B, cap] = sigmoid(s) (a monotone score, not a calibrated probability), pred_ids.span_counts [B] and pred_ids.span_types,
so Estimator.predict returns them as 'pred_spans' and InferHelper returns nested entities."""
import torch

from .. import autodiff, ops, variables
from ..data import mrc
from ..tools import layer as L
from . import _blocks as nn

SCOPE = 'global_pointer_logits'        # contains 'logit': the head's LR group and the AdamW bias exclusion
HEAD = ops.GP_HEAD                     # D = 64, the paper's default
MAX_SEQ_LEN = 512                      # ner_gp_*: i, j <= 510 fit the span key


def check_supported(params, table):
    """ValueError before any launch for a shape the GlobalPointer kernels do not take."""
    if table.L > MAX_SEQ_LEN:
        raise ValueError(f"bert_global_pointer: max_seq_len = {table.L}: the span kernels take sentences of up to "
                         f"{MAX_SEQ_LEN} positions")
    if not 1 <= table.T <= mrc.MAX_TYPES:
        raise ValueError(f"bert_global_pointer needs 1 to {mrc.MAX_TYPES} entity types, got {table.T}")


def _variables(H, T):
    w = variables.get_variable(variables.scoped(f"{SCOPE}/kernel"), (H, T * 2 * HEAD), variables.glorot_uniform)
    b = variables.get_variable(variables.scoped(f"{SCOPE}/bias"), (T * 2 * HEAD,), variables.zeros)
    return w, b


def projection(hidden, w, b, is_training):
    """Encoder rows -> P [rows, T*2D] f32 = h W + b: ops.gemm_bf16 (bf16 operands), or ops.gemm_split_f32 for the
    fp32-accurate encoder.  TRAIN records dgrad, wgrad and the bias column sum."""
    H, N = w.shape
    store = variables.default_store()
    kname, bname = (variables.scoped(f"{SCOPE}/{n}") for n in ('kernel', 'bias'))
    x2d = hidden.reshape(-1, H).contiguous()
    if not is_training and L.BERT_PRECISION == 'fp32':
        def build_split():
            return ops.split_bf16(w.t().contiguous())
        w_hi, w_lo = store.cached(("gp_pack_split", kname), build_split)
        a_hi, a_lo = ops.split_bf16(x2d)
        return ops.gemm_split_f32(a_hi, a_lo, w_hi, w_lo, bias=b)

    def build():
        return dict(nk=ops.pack_weight_bf16(w), kn=w.to(torch.bfloat16).contiguous())
    pk = store.cached(("gp_pack", kname), build)
    x16 = getattr(hidden, 'bf16', None)
    x16 = x16.reshape(-1, H) if x16 is not None else ops.cast_pad_bf16(x2d, H)
    proj = ops.gemm_bf16(x16, pk['nk'], b, epilogue=ops.EPI_F32)
    tape = autodiff.current() if is_training else None
    if tape is not None:
        need_dx = tape.needs_grad(hidden)

        def bwd(g):
            if g is None:
                return
            if need_dx:
                dx = ops.gemm_bf16(ops.cast_bf16(g), pk['kn'], None, epilogue=ops.EPI_F32)
                tape.add_grad(hidden, dx.view(hidden.shape))
            ops.wgrad_gemm(x2d, g, out=store.grad(kname))
            ops.colsum_add(g, store.grad(bname))
        tape.record(proj, bwd)
    return proj


def span_loss(proj, hi, lo, label_ids, seq_len, type_tag, B, Lq, cu, is_training):
    """Mean multilabel span cross-entropy.  TRAIN: the loss tensor with its backward (scores recomputed, then the
    transposed RoPE) recorded; EVAL / PREDICT: a variables.Deferred (targets and loss run only when it is fetched)."""
    tape = autodiff.current() if is_training else None
    if tape is None:
        return variables.Deferred(
            lambda: ops.gp_loss_fwd(hi, lo, seq_len, ops.gp_targets(label_ids, seq_len, type_tag), Lq, cu)[0])
    span_end = ops.gp_targets(label_ids, seq_len, type_tag)
    loss, lse = ops.gp_loss_fwd(hi, None, seq_len, span_end, Lq, cu)

    def bwd(g):
        d_rot = ops.gp_loss_bwd(hi, seq_len, span_end, lse, Lq, 1.0, cu)
        tape.add_grad(proj, ops.gp_rope_bwd(d_rot, B, Lq, cu))
    tape.record(loss, bwd)
    return loss


def build_graph(features, labels, params, is_training):
    nn.refuse_label_mask(features, 'bert_global_pointer')
    table = mrc.type_table(params)
    check_supported(params, table)
    B, Lq = features['token_ids'].shape
    hidden = nn.bert_sequence(features, params, is_training)    # packed rows in PREDICT / EVAL, [B, L, H] in TRAIN
    pack = getattr(hidden, 'pack', None)
    cu = pack.cu_seqlens if pack is not None else None
    w, b = _variables(hidden.shape[-1], table.T)
    proj = projection(hidden, w, b, is_training)
    split = not is_training and L.BERT_PRECISION == 'fp32'
    hi, lo = ops.gp_rope(proj, B, Lq, table.T, cu, split=split)
    seq_len = features['seq_len']
    loss = None
    if features.get('label_ids') is not None:
        loss = span_loss(proj, hi, lo, features['label_ids'], seq_len, table.type_tag, B, Lq, cu, is_training)
    pred_ids = ops.gp_decode(hi, lo, seq_len, table.type_tag, table.o_tag, table.cls_tag, table.sep_tag, Lq, cu)
    pred_ids.span_types = table.names
    return loss, pred_ids


# bert_ce's recipe: the head's name contains 'logit' (diff_lr_times, the AdamW bias exclusion)
TRAIN_PARAMS = nn.hyper(diff_lr_times={'logit': 500})
