# -*-coding:utf-8 -*-
"""`lattice_lstm_crf`: Lattice LSTM NER (Zhang & Yang, ACL 2018, "Chinese NER Using Lattice LSTM"), the baseline of the
SoftLexicon paper the word-enhance plugins restate.  The reference has no lattice plugin: the definition below restates
the paper and its public implementation, and the tests pin it.

char ids -> frozen char table -> dropout -> bidirectional lattice LSTM -> dropout -> logits -> CRF.

Lexicon input (LatticeProc): for each start character b, up to Kw = max_lattice_words vocabulary words of 2..10
characters matching at [b, b + n), lattice_ids / lattice_lens [B, L * Kw].

Forward direction, hidden size H, zero initial state; x_t the char embedding:
    [i; o; g] = W_ih x_t + W_hh h_{t-1} + b          i, o sigmoid, g tanh
    no word ends at t:  c_t = (1 - i) c_{t-1} + i g    (the coupled gate of the public code)
    else, for each word w ending at t:  a_w = sigmoid(W_ax x_t + W_ac c^w + b_a),
          c_t = (e^i g + sum_w e^{a_w} c^w) / (e^i + sum_w e^{a_w})
    h_t = o tanh(c_t)
    word cell of each word w starting at t (x^w its embedding):  [f; i^w; g^w] = W_wih x^w + W_whh h_t + b_w,
          c^w = sigmoid(f) c_t + sigmoid(i^w) tanh(g^w)     (merged at the word's last character)
The backward direction runs the same recurrence right to left: word cells at the word's last character, merged at its
first.  Positions t >= seq_len output 0.  Output [fw | bw].

Variables: lattice_layer/{fw,bw}/{char_cell,word_cell,alpha}/{kernel,bias} (TF-style [input; hidden] kernels),
word_enhance/lattice_word_embedding (trainable, initialised from params['word_embedding']), logits, crf_layer/transitions.
"""
import torch

from .. import autodiff, ops, variables
from ..tools import layer as L
from . import _blocks as nn

WORD_TABLE = 'word_enhance/lattice_word_embedding'


def build_graph(features, labels, params, is_training):
    if str(params['cell_type']).lower() != 'lstm' or int(params['cell_size']) != 1:
        raise ValueError("lattice_lstm_crf is one bidirectional lattice LSTM layer: cell_type='lstm', cell_size=1")
    input_ids = features['token_ids']
    B, Lq = input_ids.shape
    Kw = int(params.get('max_lattice_words', 4))
    lat_ids = features['lattice_ids'].reshape(B * Lq, Kw)
    lat_len = features['lattice_lens'].reshape(B, Lq * Kw)
    rate = params['embedding_dropout']
    init = params['word_embedding']
    table = variables.get_variable(WORD_TABLE, tuple(init.shape), variables.constant(init))

    chars = L.dropout(ops.embedding_lookup(nn.device_constant(params, 'embedding'), input_ids), rate, is_training)
    # slot embeddings: the SoftLexicon gather at G = Kw groups of S = 1 slot, weight 1 on slots of a plausible length
    filled = ((lat_len >= 2) & (lat_len <= 10)).to(torch.float32).reshape(B * Lq, Kw)
    words = ops.softlexicon_pool(table, lat_ids, filled, Kw, 1)                  # [B*L, Kw*Ew]
    tape = autodiff.current() if is_training else None
    if tape is not None:
        store = variables.default_store()

        def pool_bwd(g):
            if g is not None:
                ops.softlexicon_pool_bwd(store.grad(WORD_TABLE), lat_ids, filled, g.contiguous(), Kw, 1)
        tape.record(words, pool_bwd)
    words = L.dropout(words, rate, is_training)
    hidden = L.lattice_lstm(chars, words, lat_len, params['hidden_units_list'][0], features['seq_len'], is_training)
    hidden = L.dropout(hidden, rate, is_training)
    return nn.crf_head(hidden, features, params, is_training)


TRAIN_PARAMS = nn.hyper(
    dict(cell_type='lstm', cell_size=1, hidden_units_list=[100],     # the paper's 200, split over the two directions
         keep_prob_list=[1], rnn_activation='tanh'),
    lr=0.0015,
    decay_rate=0.95,
    embedding_dropout=0.5,
    early_stop_ratio=1,
)
