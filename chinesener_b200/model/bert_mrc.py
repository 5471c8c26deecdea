"""`bert_mrc`: MRC-style NER (the reference's mrc/ framework, restated; not pinned to it).  Each sentence becomes T query /
context pairs `[CLS] query_t [SEP] sentence [SEP]`, one per entity type (data/mrc.py), built on the device by
ner_mrc_pairs; BertModel runs over the pairs, a 3-unit label projection 'logits' (O, B, I) reads each pair at the
sentence's positions, trained with the masked token cross-entropy of tools/loss.py over [B*T, L, 3].  ner_mrc_merge
folds the T per-type predictions back into one tag sequence of the dataset's tag space (the highest-scoring claiming type
wins), so evaluation, prediction pickles and InferHelper see an ordinary tagger.

PREDICT / EVAL run the packed encoder; the pair token count comes from the host counts Estimator.to_device attaches to
the mask, so the graph has no device-to-host synchronisation.  TRAIN uses the packed training encoder, whose output keeps
the padded pair layout; the alignment gather and its gradient (a scatter) use ner_gather_rows / ner_scatter_rows."""
from .. import autodiff, ops
from ..data import mrc
from ..tools import layer as L
from ..tools.loss import cross_entropy_loss
from . import _blocks as nn

MRC_CLASSES = 3              # O, B, I of one entity type


def sentence_rows(hidden, align, n_pairs, max_seq_len, is_training):
    """Encoder output of the pairs -> [B*T, L, H] rows at the sentences' positions (row align[p*L + s] of the padded pair
    layout).  PREDICT / EVAL read the bf16 copy (what the label projection consumes) and put packed rows back in the padded
    pair layout first; TRAIN gathers the f32 output and records the scatter that returns the gradient."""
    src = hidden if is_training else getattr(hidden, 'bf16', hidden)
    H = src.shape[-1]
    src = src.reshape(-1, H)
    pack = getattr(hidden, 'pack', None)
    if pack is not None:
        src = ops.scatter_rows(src, pack.tok_src, pack.B * pack.L)
    rows = ops.gather_rows(src, align, n_pairs * max_seq_len).view(n_pairs, max_seq_len, H)
    tape = autodiff.current() if is_training else None
    if tape is not None:
        n_src = src.shape[0]

        def bwd(g):
            if g is not None:
                tape.add_grad(hidden, ops.scatter_rows(g.reshape(-1, H).contiguous(), align, n_src).view(hidden.shape))
        tape.record(rows, bwd)
    return rows


def build_graph(features, labels, params, is_training):
    nn.refuse_label_mask(features, 'bert_mrc')
    table = mrc.device_table(params)
    B, max_seq_len = features['token_ids'].shape
    pairs = ops.mrc_pairs(features['token_ids'], features['seq_len'], table.query_ids, table.query_len, table.type_tag,
                          table.L2, table.sep_id, label_ids=features.get('label_ids'))
    n_tokens = table.pair_tokens(features['mask'])
    if n_tokens is not None:
        pairs['mask'].total_tokens = n_tokens
    pair_features = {'token_ids': pairs['ids'], 'mask': pairs['mask'], 'segment_ids': pairs['segment_ids']}
    hidden = nn.bert_sequence(pair_features, params, is_training)
    rows = sentence_rows(hidden, pairs['align'], B * table.T, max_seq_len, is_training)
    logits = L.dense(rows, units=MRC_CLASSES, name='logits', is_training=is_training)
    loss = cross_entropy_loss(logits, pairs['labels'], pairs['seq_len'], max_seq_len, is_training)
    pred_ids = ops.mrc_merge(logits, features['seq_len'], table.type_tag, table.o_tag, table.cls_tag, table.sep_tag)
    return loss, pred_ids


# bert_ce's recipe (the reference's mrc/ parameters are not in this repository: unpinned)
TRAIN_PARAMS = nn.hyper(diff_lr_times={'logit': 500})
