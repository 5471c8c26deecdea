# -*-coding:utf-8 -*-
"""`transformer_crf_bichar` (reference model/transformer_crf_bichar.py:8-68, SURVEY §8(f) rank 4):
character + bi-character embedding -> projection + sinusoidal absolute positions -> transformer encoder -> CRF."""
import numpy as np
import torch

from .. import autodiff, ops
from ..tools.layer import crf_decode, crf_layer, dense, dropout
from ..tools.transformer.encoder import transformer_encoder
from ..tools.transformer.modules import embedding_project, sinusoidal_positional_encoding
from . import _blocks as nn
from .bilstm_crf import _const_table

_pos_cache = {}


def _pos_table(d_model, L, device):
    key = (d_model, L, str(device))
    t = _pos_cache.get(key)
    if t is None:
        t = _pos_cache[key] = torch.from_numpy(sinusoidal_positional_encoding(d_model, np.arange(L))).to(device).contiguous()
    return t


def build_graph(features, labels, params, is_training):
    """
    char + bichar embedding (+ absolute position encoding) -> transformer encoder -> CRF
    """
    input_ids = features['token_ids']
    bichar_ids = features['bichar_ids']
    label_ids = features['label_ids']
    seq_len = features['seq_len']
    B, L = input_ids.shape

    char_table = _const_table(params, 'embedding')
    bichar_table = _const_table(params, 'bichar_embedding')
    Ec, Eb = char_table.shape[1], bichar_table.shape[1]
    embedding = torch.empty((B * L, Ec + Eb), dtype=torch.float32, device=input_ids.device)
    ops.embedding_lookup(char_table, input_ids, out=embedding)
    ops.embedding_lookup(bichar_table, bichar_ids, out=embedding, col_offset=Ec)
    projected = embedding_project(embedding, params['d_model'], is_training=is_training)
    # embedding += get_pos_embedding(...): the same [L, d_model] table for every sentence (reference modules.py:200-206)
    pos = _pos_table(params['d_model'], params['max_seq_len'], input_ids.device)
    embedding = (projected.view(B, L, -1) + pos[None, :L]).view(B * L, -1)
    tape = autodiff.current() if is_training else None
    if tape is not None and tape.needs_grad(projected):
        tape.record(embedding, lambda g: tape.add_grad(projected, g) if g is not None else None)
    embedding = dropout(embedding, params['embedding_dropout'], is_training, seed=1234)

    transformer_output = transformer_encoder(encoder_input=embedding if is_training else embedding.view(B, L, -1),
                                             seq_len=seq_len, max_seq_len=params['max_seq_len'],
                                             encode_layers=params['encode_layers'], num_head=params['num_head'],
                                             dropout_rate=params['dropout_rate'], ffn_hidden=params['ffn_hidden'],
                                             is_training=is_training)
    transformer_output = dropout(transformer_output, params['dropout_rate'], is_training, seed=1234)
    if is_training:
        out2d = transformer_output
        transformer_output = out2d.view(B, L, -1)
        tape.record(transformer_output, lambda g: tape.add_grad(out2d, g.reshape(out2d.shape)) if g is not None else None)

    logits = dense(transformer_output, units=params['label_size'], name='logits', is_training=is_training)

    trans, log_likelihood = crf_layer(logits, label_ids, seq_len, params['label_size'], is_training,
                                      label_mask=features.get('label_mask'))
    pred_ids = crf_decode(logits, trans, seq_len, params['idx2tag'], is_training)
    crf_loss = (-log_likelihood).mean()

    return crf_loss, pred_ids


# MSRA-sized encoder, kept small as in the reference (its comparison point is FLAT)
TRAIN_PARAMS = nn.hyper(
    dict(num_head=8, d_model=160, ffn_hidden=320, encode_layers=2, batch_size=16, wramup_ratio=0.1, epochs=100),
    lr=0.001,
    decay_rate=0.95,
    embedding_dropout=0.3,
    dropout_rate=0.2,         # transformer sub-layer dropout
    early_stop_ratio=2,
)
