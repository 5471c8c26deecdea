"""`bert_mrc_span`: span-pointer MRC NER, the model of Li et al., "A Unified MRC Framework for Named Entity Recognition"
(ACL 2020), restated over bert_mrc's pairs (the reference's mrc/archive.py is not in this repository: not pinned to it).

Pairs, queries, encoder and sentence alignment are bert_mrc's (ner_mrc_pairs, nn.bert_sequence, sentence_rows): rows
[P = B*T, L, H].  Three heads read them:
  * 'start_logits' and 'end_logits', each a 2-class dense layer trained with the masked token cross-entropy over the pair's
    seq_len, as bert_mrc trains its 3-class head;
  * 'span_logits', the match head over every (start i, end j) pair:
        z[p,i,j] = w2 . drop(GELU_tanh(U[p,i] + V[p,j] + b1)) + b2,   [U | V] = rows . [W1[0:H] | W1[H:2H]]
    W1 = classifier1/kernel [2H, I], b1 = classifier1/bias [I], w2 = classifier2/kernel [I, 1], b2 = classifier2/bias [1],
    I = params['mrc_span_hidden'], dropout keep 1 - params['mrc_dropout'] in TRAIN only.
The U | V projection is one ops.gemm_bf16 with W1 re-packed as [2I, H] once per store version; everything after it is
csrc/mrc_span.cu: the targets from the per-type BIO labels, the match logits with the BCE loss averaged over every candidate
(1 <= i <= j <= seq_len - 2) of the batch and its backward, and the decode.  loss = CE_start + CE_end + BCE.

pred_ids [B, L] is in the dataset's tag space (evaluation, pickles and main.py see an ordinary tagger): the greedy
non-overlapping projection of the spans.  The overlapping and nested spans themselves ride along on it as
pred_ids.spans [B, cap] (ner_extract_spans' word start | end_exclusive << 12 | type << 24, type = index in the MrcTable's
names), pred_ids.span_probs [B, cap] and pred_ids.span_counts [B]."""
import torch

from .. import autodiff, ops, variables
from ..data import mrc
from ..tools import layer as L
from ..tools.loss import cross_entropy_loss
from . import _blocks as nn
from .bert_mrc import TRAIN_PARAMS as MRC_TRAIN_PARAMS
from .bert_mrc import sentence_rows

SCOPE = 'span_logits'
MAX_SEQ_LEN = 511            # ner_mrc_span_*: the pair bound
MAX_HIDDEN = 4096


def check_supported(params, table):
    """ValueError before any launch for a shape the span kernels do not take (T <= 32 is mrc.entity_types' check)."""
    I = int(params['mrc_span_hidden'])
    if I % 32 != 0 or not 32 <= I <= MAX_HIDDEN:
        raise ValueError(f"bert_mrc_span: mrc_span_hidden = {I}: the match head takes a multiple of 32 up to {MAX_HIDDEN}")
    if table.L > MAX_SEQ_LEN:
        raise ValueError(f"bert_mrc_span: max_seq_len = {table.L}: the span kernels take sentences of up to {MAX_SEQ_LEN} "
                         "positions")
    keep = 1.0 - float(params['mrc_dropout'])
    if not 0.0 < keep <= 1.0:
        raise ValueError(f"bert_mrc_span: mrc_dropout = {params['mrc_dropout']} must be in [0, 1)")
    return I, keep


def _variables(H, I):
    g = lambda n, shape, init: variables.get_variable(variables.scoped(f"{SCOPE}/{n}"), shape, init)
    w1 = g('classifier1/kernel', (2 * H, I), variables.glorot_uniform)
    b1 = g('classifier1/bias', (I,), variables.zeros)
    w2 = g('classifier2/kernel', (I, 1), variables.glorot_uniform)
    b2 = g('classifier2/bias', (1,), variables.zeros)
    return w1, b1, w2, b2


def span_projection(rows, w1, is_training):
    """rows [P, L, H] -> U | V [P*L, 2I] f32 on the tensor cores.  TRAIN records dgrad and wgrad of W1."""
    P, Lq, H = rows.shape
    I = w1.shape[1]
    store = variables.default_store()
    kname = variables.scoped(f"{SCOPE}/classifier1/kernel")

    def build():
        wcat = torch.cat([w1[:H], w1[H:]], dim=1).contiguous()              # [H, 2I]
        return dict(nk=ops.pack_weight_bf16(wcat), kn=wcat.to(torch.bfloat16).contiguous())
    pk = store.cached(("mrc_span_pack", kname), build)
    x2d = rows.reshape(P * Lq, H)
    x16 = x2d if x2d.dtype == torch.bfloat16 else ops.cast_pad_bf16(x2d.contiguous(), H)
    uv = ops.gemm_bf16(x16, pk['nk'], None, epilogue=ops.EPI_F32)
    tape = autodiff.current() if is_training else None
    if tape is not None:
        need_dx = tape.needs_grad(rows)

        def bwd(g):
            if g is None:
                return
            if need_dx:
                dx = ops.gemm_bf16(ops.cast_bf16(g), pk['kn'], None, epilogue=ops.EPI_F32)
                tape.add_grad(rows, dx.view(P, Lq, H))
            dw = ops.wgrad_gemm(x2d, g)                                         # [H, 2I]
            gk = store.grad(kname)
            gk[:H] += dw[:, :I]
            gk[H:] += dw[:, I:]
        tape.record(uv, bwd)
    return uv


def match_loss(uv, b1, w2, b2, pair_seq_len, span_end, L_sent, keep, is_training):
    """Mean BCE of the match logits over the batch's candidates.  TRAIN: the loss tensor, its backward recorded (dropout
    keep / seed regenerated there); EVAL / PREDICT: a variables.Deferred, evaluated only when the loss is fetched."""
    tape = autodiff.current() if is_training else None
    if tape is None:
        return variables.Deferred(lambda: ops.mrc_span_match_fwd(uv, b1, w2, b2, pair_seq_len, L_sent, span_end)[1])
    store = variables.default_store()
    store.dropout_calls += 1
    seed = (1234 * 1000003 + store.global_step) * 1009 + store.dropout_calls
    z, loss = ops.mrc_span_match_fwd(uv, b1, w2, b2, pair_seq_len, L_sent, span_end, keep, seed)
    names = [variables.scoped(f"{SCOPE}/{n}") for n in ('classifier1/bias', 'classifier2/kernel', 'classifier2/bias')]

    def bwd(g):
        d_uv, d_b1, d_w2, d_b2 = ops.mrc_span_match_bwd(uv, z, b1, w2, pair_seq_len, span_end, 1.0, keep, seed)
        store.grad(names[0]).add_(d_b1)
        store.grad(names[1]).view(-1).add_(d_w2)
        store.grad(names[2]).add_(d_b2)
        tape.add_grad(uv, d_uv)
    tape.record(loss, bwd)
    return loss


def build_graph(features, labels, params, is_training):
    nn.refuse_label_mask(features, 'bert_mrc_span')
    table = mrc.device_table(params)
    I, keep = check_supported(params, table)
    B, max_seq_len = features['token_ids'].shape
    pairs = ops.mrc_pairs(features['token_ids'], features['seq_len'], table.query_ids, table.query_len, table.type_tag,
                          table.L2, table.sep_id, label_ids=features.get('label_ids'))
    n_tokens = table.pair_tokens(features['mask'])
    if n_tokens is not None:
        pairs['mask'].total_tokens = n_tokens
    pair_features = {'token_ids': pairs['ids'], 'mask': pairs['mask'], 'segment_ids': pairs['segment_ids']}
    hidden = nn.bert_sequence(pair_features, params, is_training)
    rows = sentence_rows(hidden, pairs['align'], B * table.T, max_seq_len, is_training)
    start_logits = L.dense(rows, units=2, name='start_logits', is_training=is_training)
    end_logits = L.dense(rows, units=2, name='end_logits', is_training=is_training)
    w1, b1, w2, b2 = _variables(rows.shape[-1], I)
    uv = span_projection(rows, w1, is_training)
    loss = None
    if pairs['labels'] is not None:
        start_y, end_y, span_end = ops.mrc_span_targets(pairs['labels'], pairs['seq_len'])
        loss = (cross_entropy_loss(start_logits, start_y, pairs['seq_len'], max_seq_len, is_training)
                + cross_entropy_loss(end_logits, end_y, pairs['seq_len'], max_seq_len, is_training)
                + match_loss(uv, b1, w2, b2, pairs['seq_len'], span_end, max_seq_len, keep, is_training))
    pred_ids = ops.mrc_span_decode(start_logits, end_logits, uv, b1, w2, b2, features['seq_len'], table.type_tag,
                                   table.o_tag, table.cls_tag, table.sep_tag)
    pred_ids.span_types = table.names
    return loss, pred_ids


# bert_mrc's recipe: every head name contains 'logit' (diff_lr_times, the AdamW bias exclusion), plus the match head's size
# (the paper's classifier_intermediate_hidden_size) and its dropout
TRAIN_PARAMS = dict(MRC_TRAIN_PARAMS, mrc_span_hidden=1024, mrc_dropout=0.1)
