"""Shared pieces of the plugin graphs.  Every plugin keeps the reference contract — `build_graph(features, labels, params,
is_training) -> (loss, pred_ids)` plus a module-level `TRAIN_PARAMS` — and composes these blocks; the blocks call the
reference-shaped layer functions of `tools/layer.py`, which hold the kernels."""
import numpy as np
import torch

from .. import autodiff, ops, variables
from ..config import TRAIN_PARAMS as BASE_TRAIN_PARAMS
from ..tools import layer as L

SOFTWORD_TABLE = 'word_enhance/softword_embedding'
SOFTWORD_LABELS = 5                  # softword: none/[PAD], B, M, E, S; ex_softword: B, M, E, S, None


def hyper(*groups, **overrides):
    """TRAIN_PARAMS of a plugin: the shared defaults, then each group dict, then keyword overrides."""
    out = dict(BASE_TRAIN_PARAMS)
    for g in groups:
        out.update(g)
    out.update(overrides)
    return out


def device_constant(params, key):
    """A non-trainable numpy table of `params` (pretrained embeddings): one cached device copy per params dict."""
    cache = params.setdefault('_device_consts', {})
    if key not in cache:
        cache[key] = torch.as_tensor(params[key], dtype=torch.float32).cuda().contiguous()
    return cache[key]


def bert_sequence(features, params, is_training, packed=True):
    """BertModel sequence output for the batch (reference tools/layer.py:63-81).  packed=False keeps the padded layout for
    plugins whose next layer reads [PAD] positions."""
    args = (features['token_ids'], features['mask'], features['segment_ids'], params['pretrain_dir'],
            params['embedding_dropout'], is_training)
    if packed:
        return L.pretrain_bert_embedding(*args)
    keep, L.PACK_SEQUENCES = L.PACK_SEQUENCES, False
    try:
        return L.pretrain_bert_embedding(*args)
    finally:
        L.PACK_SEQUENCES = keep


def recurrent(x, features, params, is_training):
    """The bidirectional LSTM block configured by the plugin's RNN hyper-parameters."""
    return L.bilstm(x, params['cell_type'], params['rnn_activation'], params['hidden_units_list'], params['keep_prob_list'],
                    params['cell_size'], features['seq_len'], params['dtype'], is_training)


def bilstm_crf_tail(embedding, features, params, is_training):
    """bilstm_crf's graph after the embedding: dropout -> BiLSTM -> dropout -> label projection -> CRF."""
    rate = params['embedding_dropout']
    hidden = recurrent(L.dropout(embedding, rate=rate, is_training=is_training, seed=1234), features, params, is_training)
    hidden = L.dropout(hidden, rate=rate, is_training=is_training, seed=1234)
    return crf_head(hidden, features, params, is_training)


def segmentation_embedding(features, params, is_training, ids=None, weights=None):
    """[W[ids] (softword) or weights @ W (ex_softword) | frozen character embedding] -> [B, L, 5 + Ec], both pieces
    written into one buffer.  W is the trainable [5, 5] `word_enhance/softword_embedding`, identity at initialisation;
    TRAIN records its gradient, read from the first 5 columns of the buffer's gradient by ner_small_table_grad."""
    input_ids = features['token_ids']
    B, Lq = input_ids.shape
    char_table = device_constant(params, 'embedding')
    n = SOFTWORD_LABELS
    table = variables.get_variable(SOFTWORD_TABLE, (n, n), variables.constant(np.eye(n, dtype=np.float32)))
    embedding = torch.empty((B, Lq, n + char_table.shape[1]), dtype=torch.float32, device=input_ids.device)
    if weights is not None:
        weights = weights.reshape(B, Lq, n)
        ops.multihot_embed(table, weights, out=embedding)
    else:
        ops.embedding_lookup(table, ids, out=embedding)
    ops.embedding_lookup(char_table, input_ids, out=embedding, col_offset=n)
    tape = autodiff.current() if is_training else None
    if tape is not None:
        store = variables.default_store()

        def bwd(g):
            if g is not None:
                ops.small_table_grad(store.grad(SOFTWORD_TABLE), g.contiguous(), ids=ids, weights=weights)
        tape.record(embedding, bwd)
    return embedding


def crf_head(hidden, features, params, is_training, name='logits'):
    """Label projection + CRF: -> (mean negative log-likelihood, Viterbi tags).  A batch with a `label_mask` feature
    (partially annotated sentences) is trained and evaluated with the partial-annotation CRF loss."""
    n_tags, lengths = params['label_size'], features['seq_len']
    emissions = L.dense(hidden, units=n_tags, name=name, is_training=is_training)
    transitions, log_lik = L.crf_layer(emissions, features['label_ids'], lengths, n_tags, is_training,
                                       label_mask=features.get('label_mask'))
    tags = L.crf_decode(emissions, transitions, lengths, params['idx2tag'], is_training)
    return (-log_lik).mean(), tags


def refuse_label_mask(features, plugin):
    """Plugins that read label_ids as complete gold labels cannot train on partially annotated batches: refuse one
    before anything is launched."""
    if features.get('label_ids') is not None and features.get('label_mask') is not None:
        raise ValueError(f"{plugin} cannot use partial labels (a 'label_mask' feature); train it on fully labelled "
                         f"data, or use a CRF plugin")
